"""Parity gates of SURVEY.md section 8d -- TEST INFRASTRUCTURE (used by tests/ and by bench.py's untimed
in-run parity leg; never by the product path).

`run_gates` replays ONE iteration of the recipe through the reference (oracle/refpath.py: the unmodified
reference MEX targets in oracle/_ref + the numpy restatement of the M-only psdscale) on the same inputs a
`sedumi_b200.device.HotPath` has just processed, and compares what both produced:

    ADA, absd            <= 1e-10 relative (Frobenius)          getada1-3
    L (factor), d        <= 1e-10 (Frobenius / infinity norm)   blkchol; identical skip and add index sets
    y (search direction) <= 1e-8  relative                      fwblkslv, ./d, bwblkslv
    udsqr, psdscale, frames (psdframeit), urotorder (bit-exact u/perm/gjc), givensrot  <= 1e-10

It also reports how long the reference spent inside its mexFunctions (+ numpy psdscale) for that iteration, so
that the same CPU work serves as bench.py's `cpu_baseline` sample.
"""
from __future__ import annotations

import ctypes as C
import time

import numpy as np

import refpath
import replay

TOL = {"d_dense": 1e-10, "ADA": 1e-10, "absd": 1e-10, "L": 1e-10, "d": 1e-10, "y": 1e-8, "udsqr": 1e-10, "psdscale": 1e-10,
       "frame": 1e-10, "givensrot": 1e-10}


def _rel(a, b, ord=None):
    a = np.asarray(a, dtype=float).ravel()
    b = np.asarray(b, dtype=float).ravel()
    nb = np.linalg.norm(b, ord)
    return float(np.linalg.norm(a - b, ord) / (nb if nb > 0 else 1.0))


def device_outputs(hp, S, nnzL):
    """What the device holds after hp.iteration(...): host copies."""
    from sedumi_b200 import device
    L = device.lib()
    hp.sync()
    t = hp.torch
    Lcsc = t.empty(max(nnzL, 1), dtype=t.float64, device=hp.dev)
    device.check(L.sb200_chol_rect_to_csc_dev(hp.chol, C.c_void_p(hp.Lrect.data_ptr()), C.c_void_p(hp.flag.data_ptr()),
                                              C.c_void_p(Lcsc.data_ptr())), "rect_to_csc")
    hp.sync()
    n2 = hp.lenud
    out = dict(ADA=hp.ADA.cpu().numpy()[:S.ADA.nnz], absd=hp.absd.cpu().numpy()[:S.m], L=Lcsc.cpu().numpy()[:nnzL],
               d=hp.dvec.cpu().numpy()[:S.m], flag=hp.flag.cpu().numpy()[:S.m], y=hp.y.cpu().numpy().T.copy())
    if n2:
        out.update(udsqr=hp.udsqr.cpu().numpy()[:n2], psd=hp.psd_y.cpu().numpy()[:n2], frame=hp.psd_f.cpu().numpy()[:n2],
                   u=hp.u_new.cpu().numpy()[:n2], perm=hp.perm_new.cpu().numpy()[:hp.sumn], gjc=hp.gjc.cpu().numpy()[:hp.sumn],
                   q=hp.psd_z.cpu().numpy()[:n2])
    return out


def reference_iteration(S, d, rhs, psd_x, frames, nsolve, npsd, *, S_local=None, d_local=None, tail=True):
    """What the gates compare against: one iteration of the recipe through the reference, as a dict of arrays
    (ADA and L values, absd, d, skip/add columns, y, and the PSD outputs of this rank's cone)."""
    Sl = S_local if S_local is not None else S
    dl = d_local if d_local is not None else d
    R = refpath.RefHotPath(S)
    t_np = 0.0
    m0 = R.mex.mex_seconds()
    udsqr, ADA, absd = R.assemble(d)
    from sedumi_b200.host import setup as hsetup
    LL, Ld, skip, add = R.mex.blkchol(hsetup.L_for_mex(dict(S.L)), ADA, R.pars, absd, nlhs=4)
    Lref = R.factor(ADA, absd)
    y = None
    dense = getattr(S, "dense", None)
    out = {}
    if dense is not None and len(dense.cols):            # deninfac.m:57-79 on the reference's own MEX files
        DC = refpath.DenseColumnRef(S, Lref)
        LAD, Ld0, sym, smult = DC.inputs(d, np.asarray(Ld, dtype=float).ravel().copy())
        Lden, dden = R.mex.dpr1fact(LAD, Ld0.reshape(-1, 1), sym, smult, 5e2, nlhs=2)
        Lden.update(dz=sym["dz"], first=sym["first"], perm=sym["perm"])
        Lm = hsetup.L_for_mex({k: Lref[k] for k in ("perm", "L", "xsuper", "tmpsiz")})
        for _ in range(nsolve):
            y = R.mex.bwblkslv(Lm, R.mex.bwdpr1(Lden, R.mex.fwdpr1(Lden, R.mex.fwblkslv(Lm, rhs)) / np.asarray(dden).reshape(-1, 1)))
        out["d_dense"] = np.asarray(dden, dtype=float).ravel()
    else:
        for _ in range(nsolve):
            y = R.solve(Lref, rhs)
    out.update(ADA=ADA.data, absd=np.asarray(absd, dtype=float).ravel(), L=LL.data, Ljc=np.asarray(LL.indptr),
               d=np.asarray(Ld, dtype=float).ravel(), skip=np.asarray(skip.indices), add=np.asarray(add.indices),
               y=np.asarray(y, dtype=float))
    if int((np.asarray(Sl.K["s"]) ** 2).sum()):
        Rl = R if Sl is S else refpath.RefHotPath(Sl)
        out["udsqr"] = np.asarray(udsqr if Sl is S else Rl.mex.invcholfac(dl["u"], Rl.Km, dl["perm"]), dtype=float).ravel()
        ps = None
        t1 = time.perf_counter()
        for i in range(npsd):
            ps = Rl.psdscale(dl, psd_x, i & 1)
        t_np += time.perf_counter() - t1
        if ps is not None:
            out["psd"] = np.asarray(ps, dtype=float).ravel()
        if tail and ps is not None:
            rt = Rl.scaling_tail(dl, frames[0], frames[1], np.asarray(ps).ravel())
            out.update(frame=np.asarray(rt["frame"], dtype=float).ravel(), q=np.asarray(rt["q"], dtype=float).ravel(),
                       u=np.asarray(rt["u"], dtype=float).ravel(), perm=np.asarray(rt["perm"], dtype=float).ravel(),
                       gjc=np.asarray(rt["gjc"], dtype=float).ravel())
    out["ref_seconds"] = np.array([(R.mex.mex_seconds() - m0) + t_np])
    return out


def _rel_to(a, b, ord=None):
    """_rel against a reference value that may be kept as a sketch (oracle/replay.py)."""
    if isinstance(b, replay.Sketch):
        assert ord is None
        return float(b.error_norm(np.asarray(a, dtype=float).ravel()) / (b.norm if b.norm > 0 else 1.0))
    return _rel(a, b, ord)


def _equal(a, b):
    if isinstance(b, replay.Sketch):
        return b.matches(np.asarray(a, dtype=float).ravel())
    return bool(np.array_equal(np.asarray(a, dtype=float).ravel(), np.asarray(b, dtype=float).ravel()))


def run_gates(hp, S, d, rhs, psd_x, frames, nsolve, npsd, *, S_local=None, d_local=None, colmask=None, tail=True):
    """Compare the state `hp` holds after hp.iteration(nsolve, npsd[, sharded]) with the reference.
    S/d: the FULL problem and scaling (ADA, factor, solve); S_local/d_local: this rank's cone when the PSD part is
    sharded (owner computes), else None; colmask: columns of the factor this rank answers for (sharded) or None.
    Inside a test the reference iteration is the recorded one (replay.result).
    Returns {"ok": bool, "err": {...}, "tol": {...}, "skip_equal", "add_equal", "ref_seconds", ...}."""
    nnzL = int(S.L["L"].nnz)
    dev = device_outputs(hp, S, nnzL)
    w0 = time.perf_counter()
    dl = d_local if d_local is not None else d
    ref = replay.result((d, dl, rhs, psd_x, frames[0], frames[1]),
                        lambda: reference_iteration(S, d, rhs, psd_x, frames, nsolve, npsd, S_local=S_local,
                                                    d_local=d_local, tail=tail))
    err, info = {}, {}
    err["ADA"] = _rel_to(dev["ADA"], ref["ADA"])
    err["absd"] = _rel(dev["absd"], ref["absd"])
    skip, add = np.asarray(ref["skip"]).astype(np.int64), np.asarray(ref["add"]).astype(np.int64)
    if colmask is None:
        err["L"] = _rel_to(dev["L"], ref["L"])
        err["d"] = _rel(dev["d"], ref["d"], np.inf)
        sk_dev, ad_dev = np.flatnonzero(dev["flag"] == 1), np.flatnonzero(dev["flag"] == 2)
        info["skip_equal"] = bool(np.array_equal(sk_dev, skip))
        info["add_equal"] = bool(np.array_equal(ad_dev, add))
    else:                                   # sharded factor: the columns this rank answers for (its subtrees + the top)
        cols = np.flatnonzero(colmask)
        jc = np.asarray(ref["Ljc"]).astype(np.int64)
        sel = np.concatenate([np.arange(jc[c], jc[c + 1]) for c in cols]) if cols.size else np.zeros(0, dtype=np.int64)
        err["L"] = _rel(dev["L"][sel], np.asarray(ref["L"])[sel])
        err["d"] = _rel(dev["d"][cols], ref["d"][cols], np.inf)
        info["skip_equal"] = bool(np.array_equal(np.flatnonzero(dev["flag"][cols] == 1), np.flatnonzero(np.isin(cols, skip))))
        info["add_equal"] = bool(np.array_equal(np.flatnonzero(dev["flag"][cols] == 2), np.flatnonzero(np.isin(cols, add))))
        info["factor_scope"] = f"{cols.size} of {S.m} columns (this rank's subtrees + replicated top)"
    err["y"] = _rel(dev["y"], ref["y"])
    if "d_dense" in ref:
        err["d_dense"] = _rel(hp.dvec_den.cpu().numpy()[:S.m], ref["d_dense"], np.inf)
    info["nskip"], info["nadd"] = int(skip.size), int(add.size)
    if hp.lenud:
        err["udsqr"] = _rel_to(dev["udsqr"], ref["udsqr"])
        if "psd" in ref:
            err["psdscale"] = _rel_to(dev["psd"], ref["psd"])
        if "frame" in ref:
            err["frame"] = _rel_to(dev["frame"], ref["frame"])
            err["givensrot"] = _rel_to(dev["q"], ref["q"])
            info["urotorder_bit_exact"] = bool(_equal(dev["u"], ref["u"]) and
                                               np.array_equal(dev["perm"] + 1, np.asarray(ref["perm"]).astype(np.int64)) and
                                               np.array_equal(dev["gjc"], np.asarray(ref["gjc"]).astype(np.int64)))
    ok = all(err[k] <= TOL[k] for k in err) and info.get("skip_equal", True) and info.get("add_equal", True) \
        and info.get("urotorder_bit_exact", True)
    return dict(ok=bool(ok), err=err, tol={k: TOL[k] for k in err}, ref_seconds=float(np.asarray(ref["ref_seconds"]).ravel()[0]),
                ref_wall=time.perf_counter() - w0, **info)
