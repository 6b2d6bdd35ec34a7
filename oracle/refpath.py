"""The reference's per-iteration hot path, replayed on the CPU -- TEST INFRASTRUCTURE.

Drives the UNMODIFIED reference MEX targets compiled into oracle/_ref (oracle/Makefile) plus the
numpy restatement of the M-only glue (oracle/restate.py) through the call sequence of
sedumi.m:442-466 and wrapPcg.m:56-59.  Used by tests (parity oracle), by __graft_entry__.smoke()
and by bench.py's cpu_baseline / --impl reference legs -- never by the product path.
"""
from __future__ import annotations

import os
import sys

import numpy as np
import scipy.sparse as sp

_HERE = os.path.dirname(os.path.abspath(__file__))
_ROOT = os.path.dirname(_HERE)
for _p in (_ROOT, _HERE):
    if _p not in sys.path:
        sys.path.insert(0, _p)

import replay  # noqa: E402
import restate  # noqa: E402
from sedumi_b200.host import setup as hsetup  # noqa: E402

CHOL_PARS = {"canceltol": 1e-12, "maxu": 5e5, "abstol": 1e-20}      # checkpars.m:150-170


def ref_dir(debug=False) -> replay.OracleDir:
    """The reference targets, answered from tests/golden/oracle where a record exists (oracle/replay.py)."""
    return replay.OracleDir(debug)


class RefHotPath:
    """Reference call sequence on one problem (S = sedumi_b200.host.setup.HotPathSetup)."""

    def __init__(self, S, chol_pars=None, debug=False):
        self.S = S
        self.mex = ref_dir(debug)
        self.Km = S.Kmex()
        self.pars = dict(CHOL_PARS, **(chol_pars or {}))
        self.ADA0 = sp.csc_matrix((np.zeros(S.ADA.nnz), S.ADA.indices, S.ADA.indptr), shape=S.ADA.shape)

    def DAtq(self, d):
        """getDAtm.m:40-43 (no dense Lorentz blocks)."""
        S, K = self.S, self.S.K
        tr = hsetup.extractA(S.At, S.Ablkjc, 1, 2, int(K["mainblks"][0]), int(K["mainblks"][1]))
        if len(K["q"]) == 0:
            return tr
        return sp.csc_matrix(sp.diags(d["q1"]) @ tr +
                             self.mex.ddot(d["q2"], S.At, K["qblkstart"].reshape(1, -1), S.Ablkjc))

    def assemble(self, d):
        """sedumi.m:450-452: returns (udsqr, ADA, absd)."""
        S, mex = self.S, self.mex
        if len(S.K["s"]) == 0:                      # sedumi.m:446-448: the M path, restated in numpy
            import restate
            ADA, absd = restate.getada_m(S.At, S.K, d, self.DAtq(d), pattern=S.ADA)
            return np.zeros(0), ADA, absd.reshape(-1, 1)
        udsqr = mex.invcholfac(d["u"], self.Km, d["perm"])
        A1 = mex.getada1(self.ADA0, S.At, S.Ablkjc[:, 2], S.Aord["lqperm"], {"l": d["l"], "det": d["det"]},
                         S.K["qblkstart"].reshape(1, -1))
        A2 = mex.getada2(A1, {"q": self.DAtq(d)}, S.Aord, self.Km)
        ADA, absd = mex.getada3(A2, S.At, S.Ablkjc[:, 2], S.Aord, udsqr, self.Km, nlhs=2)
        return udsqr, ADA, absd

    def factor(self, ADA, absd):
        """sedumi.m:458 + deninfac.m:81-93 (no dense columns)."""
        L = dict(self.S.L)
        LL, Ld, skip, add = self.mex.blkchol(hsetup.L_for_mex(L), ADA, self.pars, absd, nlhs=4)
        L.update(L=LL, d=Ld.ravel().copy(), skip=skip, add=add)
        sk = skip.indices
        if sk.size:
            dtol = np.maximum(self.pars["canceltol"] * absd.ravel()[L["perm"].ravel().astype(int)[sk] - 1], self.pars["abstol"])
            fix = L["d"][sk] <= dtol
            L["d"][sk[fix]] = 1.0
        return L

    def solve(self, L, r):
        """wrapPcg.m:56-59 without dense columns."""
        Lm = hsetup.L_for_mex({k: L[k] for k in ("perm", "L", "xsuper", "tmpsiz")})
        p = self.mex.fwblkslv(Lm, r)
        y = p / L["d"].reshape(-1, 1)
        return self.mex.bwblkslv(Lm, y)

    def psdscale(self, d, x, transp):
        return restate.psdscale({"u": d["u"], "perm": d["perm"]}, x, self.S.K, transp)

    def scaling_tail(self, d, lab, frms, y_psd):
        """psdinvjmul -> 2 x psdframeit -> urotorder -> givensrot on the reference's own MEX
        (updtransfo.m:99-108; SURVEY 8d recipe)."""
        Km, mex = self.Km, self.mex
        z = mex.psdinvjmul(lab, frms, y_psd, Km)
        f = mex.psdframeit(lab, frms, Km)
        f = mex.psdframeit(lab, frms, Km)
        u, perm, gjc, g = mex.urotorder(d["u"], Km, 1.1, nlhs=4)
        q = mex.givensrot(gjc, g, f, Km)
        return dict(z=z, frame=f, u=u, perm=perm, gjc=gjc, g=g, q=q)

    def lorentz_streams(self, d, mu, xq, rhi, rlo, ry):
        """6 x qblkmul, 3 x ddot (dense), 1 x quadadd on the reference's MEX (SURVEY 8d recipe, sum(K.s)==0)."""
        bs = self.S.K["qblkstart"].reshape(1, -1)
        y = dd = None
        for _ in range(6):
            y = self.mex.qblkmul(mu, xq, bs)
        for _ in range(3):
            dd = self.mex.ddot(d["q2"], xq, bs)
        zhi, zlo = self.mex.quadadd(rhi, rlo, ry, nlhs=2)
        return dict(y=y, dd=dd, zhi=zhi, zlo=zlo)

    def iteration(self, d, rhs, psd_x, nsolve=4, npsdscale=12, frames=None):
        udsqr, ADA, absd = self.assemble(d)
        L = self.factor(ADA, absd)
        y = None
        for _ in range(nsolve):
            y = self.solve(L, rhs)
        ps = None
        for i in range(npsdscale if len(self.S.K["s"]) else 0):
            ps = self.psdscale(d, psd_x, i & 1)
        out = dict(udsqr=udsqr, ADA=ADA, absd=absd, L=L, y=y, psd=ps)
        if frames is not None and len(self.S.K["s"]):
            out["tail"] = self.scaling_tail(d, frames[0], frames[1], np.asarray(ps).ravel())
        return out


class DenseColumnRef:
    """Dense-column (product-form) part of the reference path for LP dense columns:
    symbcholden.m:45-55 (symbolic, via the reference's symbfwblk/incorder/finsymbden) and
    deninfac.m:57-79 (numeric: sparfwslv + dpr1fact)."""

    def __init__(self, S, L, debug=False):
        self.mex = ref_dir(debug)
        self.S = S
        dense = S.dense
        assert len(dense.q) == 0, "only LP dense columns are exercised here"
        Lm = hsetup.L_for_mex({k: L[k] for k in ("perm", "L", "xsuper", "tmpsiz")})
        self.Lm = Lm
        i1 = dense.l + 1
        LAD = self.mex.symbfwblk(Lm, sp.csc_matrix(dense.A[:, :i1 - 1]))
        perm, dz = self.mex.incorder(LAD, nlhs=2)
        self.sym = self.mex.finsymbden(LAD, perm, dz, float(i1))
        self.sym["LAD"] = LAD

    def inputs(self, d, Ld):
        """(LAD values, L.d, symLden, smult, maxu) as deninfac.m hands them to dpr1fact."""
        dense = self.S.dense
        Ad = sp.csc_matrix(dense.A)
        smult = d["l"][dense.cols[:dense.l].astype(int) - 1]
        LAD = self.mex.fwblkslv(self.Lm, Ad, self.sym["LAD"])
        return LAD, Ld, self.sym, smult.reshape(-1, 1)


def wrappcg_direct(R: "RefHotPath", L: dict, d: dict, rv, rb=None):
    """The direct step of wrapPcg.m:42-97 (no dense columns, no Lorentz cones) driven through the reference's own
    MEX solves and vecsym, with numpy for the M-only glue (Amul.m:42-56, psdscale.m) -- the parity point of the
    search direction (SURVEY 8c/8f).  Returns dict(y, dx, r, ssqrNew, ssqrdx, alpha, normr)."""
    S = R.S
    K = S.K
    l = int(K["l"])
    At = S.At
    rv = np.asarray(rv, dtype=float).ravel()
    sl = np.sqrt(np.asarray(d["l"], dtype=float).ravel())

    def D(x, transp):
        return np.r_[sl * x[:l], restate.psdscale({"u": d["u"], "perm": d["perm"]}, x, K, transp)]

    Lm = hsetup.L_for_mex({k: L[k] for k in ("perm", "L", "xsuper", "tmpsiz")})
    Ld = np.asarray(L["d"], dtype=float).reshape(-1, 1)
    dx = D(rv, 1)
    r = np.asarray(At.T @ dx).ravel()
    if rb is not None:
        r = r + np.asarray(rb, dtype=float).ravel()
    p = R.mex.fwblkslv(Lm, r.reshape(-1, 1))
    y = p / Ld
    ssq = float((p * y).sum())
    p = np.asarray(R.mex.bwblkslv(Lm, y)).ravel()
    x = np.asarray(At @ p).ravel()
    x = np.asarray(R.mex.vecsym(x.reshape(-1, 1), R.Km)).ravel()
    dx2 = D(x, 0)
    ssqrdx = float(dx2 @ dx2)
    alpha = ssq / ssqrdx
    yout = alpha * p
    dxo = rv - alpha * dx2
    x = D(dxo, 1)
    r = np.asarray(At.T @ x).ravel()
    if rb is not None:
        r = r + np.asarray(rb, dtype=float).ravel()
    return dict(y=yout, dx=dxo, r=r, ssqrNew=ssq, ssqrdx=ssqrdx, alpha=alpha, normr=float(np.abs(r).max()))
