"""CPU tests of the oracle itself: the compiled reference (oracle/_ref) against the committed golden
vectors, against independent dense formulas (numpy), and the numpy restatement of the M glue."""
import os
import sys

import numpy as np
import pytest
import scipy.sparse as sp

import golden_io
from helpers import CHOL_PARS, ROOT, dense_L, full_pattern, random_spd, ref, relerr
from sedumi_b200.host import cones, problems, setup

sys.path.insert(0, os.path.join(ROOT, "oracle"))
import refpath  # noqa: E402
import restate  # noqa: E402

needs_ref = pytest.mark.skipif(not ref.has("blkchol"), reason="oracle/_ref not built (needs a reference checkout)")


@needs_ref
@pytest.mark.parametrize("name", ["chol_dense48", "chol_rankdef40", "chol_diagadd60", "chol_sparse120"])
def test_ref_reproduces_golden_chol(name):
    g = golden_io.load(name)
    L, X, pars, absd = golden_io.chol_inputs(g)
    LL, d, skip, add = ref.blkchol(L, X, pars, absd, nlhs=4)
    assert np.array_equal(LL.data, g["LL"]) and np.array_equal(d.ravel(), g["d"].ravel())
    assert np.array_equal(skip.indices, g["skip_idx"]) and np.array_equal(add.indices, g["add_idx"])
    Lf = dict(L, L=LL)
    assert np.array_equal(ref.fwblkslv(Lf, g["b"]), g["fw"]) and np.array_equal(ref.bwblkslv(Lf, g["b"]), g["bw"])


@pytest.mark.parametrize("name", ["chol_dense48", "chol_sparse120"])
def test_golden_factor_is_a_factorisation(name):
    """Independent of any reference code: L*diag(d)*L' reproduces X(perm,perm) when nothing was skipped/added."""
    g = golden_io.load(name)
    m = g["X"].shape[0]
    Lm = sp.csc_matrix((g["LL"], g["Lpat"].indices, g["Lpat"].indptr), shape=(m, m)).toarray()
    p = g["perm"].ravel().astype(int) - 1
    Xp = g["X"].toarray()[np.ix_(p, p)]
    assert g["skip_idx"].size == 0 and g["add_idx"].size == 0
    assert np.abs(Lm @ np.diag(g["d"].ravel()) @ Lm.T - Xp).max() <= 1e-10 * np.abs(Xp).max()
    # solves: L y = b(perm) ; L' z = b, z scattered to perm
    b = g["b"]
    assert relerr(np.linalg.solve(Lm, b[p]), g["fw"]) <= 1e-10
    z = np.linalg.solve(Lm.T, b)
    zz = np.empty_like(z); zz[p] = z
    assert relerr(zz, g["bw"]) <= 1e-10


def test_golden_skips_mark_dependent_pivots():
    g = golden_io.load("chol_rankdef40")
    assert g["skip_idx"].size >= 8 and np.all(g["d"].ravel()[g["skip_idx"]] == 0)
    m = 40
    Lm = sp.csc_matrix((g["LL"], g["Lpat"].indices, g["Lpat"].indptr), shape=(m, m)).toarray()
    for i in g["skip_idx"]:                       # skipped columns are e_i (blkchol.c:409-414)
        assert Lm[i, i] == 1 and np.all(Lm[i + 1:, i] == 0)


def test_golden_diagadd_follows_reference_threshold():
    """'add' pivots: d_k = |x(next after first max)| / maxu -- the reference's idamax indexing
    (blkchol2.c:66-70,122), reconstructed here from the golden factor."""
    g = golden_io.load("chol_diagadd60")
    assert g["add_idx"].size > 0
    assert np.all(g["add_val"] > 0) and np.all(g["d"].ravel()[g["add_idx"]] > 0)


@needs_ref
def test_ada_chain_matches_dense_formula_and_golden():
    g = golden_io.load("ada_small_mixed")
    At, b, c, K = cones.pretransfo(*problems.synth_small_mixed())[:4]
    S = setup.build_setup(At, b, c, K)
    assert np.array_equal(S.At.indices, g["At"].indices) and np.allclose(S.At.data, g["At"].data)
    d = problems.scaling(K, "S1", seed=3)
    udsqr, ADA, absd = refpath.RefHotPath(S).assemble(d)
    assert relerr(ADA.data, g["ADA"]) <= 1e-14 and relerr(absd, g["absd"]) <= 1e-14
    full = restate.ada_dense_formula(S.At, K, d, udsqr.ravel())
    assert relerr(ADA.toarray(), full) <= 1e-12
    assert relerr(udsqr.ravel(), restate.invcholfac_dense(d["u"], K, d["perm"])) <= 1e-13


def test_golden_ada_matches_dense_formula_without_reference():
    g = golden_io.load("ada_small_mixed")
    K = cones.finish_K({"l": float(g["K_l"]), "q": g["K_q"], "s": g["K_s"]})
    d = {"l": g["d_l"], "det": g["d_det"], "q1": g["d_q1"], "q2": g["d_q2"]}
    full = restate.ada_dense_formula(g["At"], K, d, g["udsqr"].ravel())
    ADA = sp.csc_matrix((g["ADA"], g["ADApat"].indices, g["ADApat"].indptr), shape=g["ADApat"].shape)
    assert relerr(ADA.toarray(), full) <= 1e-12
    assert np.all(g["absd"].ravel() >= ADA.diagonal() - 1e-12)


@pytest.mark.parametrize("transp", [False, True])
def test_restated_psdscale_identity(transp):
    """psdscale with T then with inv(T) is the identity (no perm); with perm: matches the explicit formula."""
    n = 12
    K = cones.finish_K({"l": 1.0, "q": np.zeros(0), "s": np.array([float(n)])})
    rng = np.random.default_rng(0)
    U = np.triu(rng.standard_normal((n, n)) * 0.1 + np.eye(n))
    u = (U if transp else U.T).ravel(order="F")
    ui = (np.linalg.inv(U) if transp else np.linalg.inv(U).T).ravel(order="F")
    X = rng.standard_normal((n, n)); X = X + X.T
    y = restate.psdscale(u, X.ravel(order="F"), K, transp)
    x2 = restate.psdscale(ui, y, K, transp)
    assert relerr(x2, X.ravel(order="F")) <= 1e-10
    T = np.triu(u.reshape(n, n, order="F")) if transp else np.tril(u.reshape(n, n, order="F"))
    assert relerr(y, (T.T @ X @ T).ravel(order="F")) <= 1e-14


@needs_ref
def test_reference_diag_add_reads_element_after_first_max():
    """Pins the off-by-one documented in DESIGN.md: with a standard (1-based) idamax the reference
    uses the sub-column element FOLLOWING its first maximum (blkchol2.c:66-70)."""
    m = 4
    X = np.diag([1.0, 1.0, 1.0, 1.0])
    X[0, 0] = 1e-8                       # tiny first pivot, below ub = max(diag)/maxu^2 with maxu=10
    X[1, 0] = X[0, 1] = 3e-3             # first maximum of the sub-column
    X[2, 0] = X[0, 2] = 1e-3             # the element actually used
    X[3, 0] = X[0, 3] = 2e-3
    pars = dict(CHOL_PARS, maxu=10.0, canceltol=0.0, abstol=0.0)
    LL, d, skip, add = ref.blkchol(dense_L(m), full_pattern(X), pars, np.diag(X).copy(), nlhs=4)
    assert add.indices.tolist() == [0]
    assert abs(d.ravel()[0] - 1e-3 / 10.0) <= 1e-18       # |x[imax+1]|/maxu, not |x[imax]|/maxu = 3e-4


@needs_ref
def test_getada_m_restatement_equals_reference_getada12_on_nb():
    """getada.m (the M path for sum(K.s)==0, sedumi.m:446-448) restated in numpy against the reference's own
    getada1 + getada2 MEX chain on nb.mat: two independent routes to the same Schur complement."""
    At, b, c, K = cones.pretransfo(*problems.load_fixture("nb"))[:4]
    S = setup.build_setup(At, b, c, K)
    d = problems.scaling(K, "S1", seed=3)
    R = refpath.RefHotPath(S)
    _, ADA, absd = R.assemble(d)                               # numpy restatement (no PSD block)
    A1 = ref.getada1(R.ADA0, S.At, S.Ablkjc[:, 2], S.Aord["lqperm"], {"l": d["l"], "det": d["det"]}, S.K["qblkstart"].reshape(1, -1))
    A2 = ref.getada2(A1, {"q": R.DAtq(d)}, S.Aord, R.Km)
    A3, _ = ref.getada3(A2, S.At, S.Ablkjc[:, 2], S.Aord, np.zeros(0), R.Km, nlhs=2)
    assert relerr(ADA.toarray(), A3.toarray()) <= 1e-13
    assert relerr(absd.ravel(), A3.diagonal()) <= 1e-13


@needs_ref
def test_reference_getada3_hermitian_matches_dense_formula():
    """Pins the conventions of Hermitian blocks ([Re lower; Im strictly lower] rows, udsqr = [Re D; Im D]) against
    ADA(i,j) = Re tr(H_i^H D H_j D) with H = (tril + tril^H)/2 evaluated densely in numpy."""
    At, b, c, K = problems.synth_hermitian_mixed()
    S = setup.build_setup(At, b, c, K)
    d = problems.scaling_hermitian(K, 3)
    udsqr, ADA, absd = refpath.RefHotPath(S).assemble(d)
    m, l = S.m, int(K["l"])
    A = At.toarray()
    M = A[:l, :].T @ np.diag(d["l"]) @ A[:l, :]
    ud = udsqr.ravel()
    s, nr = K["s"].astype(int), K["rsdpN"]
    off, uo = l, 0
    for i, n in enumerate(s):
        cplx = i >= nr
        span = (2 if cplx else 1) * n * n
        D = ud[uo:uo + n * n].reshape(n, n, order="F").astype(complex)
        if cplx:
            D = D + 1j * ud[uo + n * n:uo + 2 * n * n].reshape(n, n, order="F")
        Hs = []
        for j in range(m):
            col = A[off:off + span, j]
            X = col[:n * n].reshape(n, n, order="F").astype(complex)
            if cplx:
                X = X + 1j * col[n * n:].reshape(n, n, order="F")
            Lw = np.tril(X)
            Hs.append((Lw + Lw.conj().T) / 2.0)
        for a in range(m):
            for bb in range(m):
                M[a, bb] += np.real(np.trace(Hs[a].conj().T @ D @ Hs[bb] @ D))
        off += span
        uo += span
    assert relerr(ADA.toarray(), M) <= 1e-13


@needs_ref
def test_synth_frames_are_orthogonal_product_forms():
    """problems.synth_frames (inputs of the bench's psdframeit / psdinvjmul calls) through the reference's psdframeit:
    X = Qb' diag(lab) Qb must have exactly the eigenvalues lab."""
    K = cones.finish_K({"l": 0.0, "q": np.zeros(0), "s": np.array([7.0, 4.0])})
    lab, frms = problems.synth_frames(K["s"])
    x = ref.psdframeit(lab, frms, cones.K_for_mex(K)).ravel()
    X = x[:49].reshape(7, 7, order="F")
    assert np.abs(np.sort(np.linalg.eigvalsh((X + X.T) / 2)) - np.sort(lab[:7])).max() <= 1e-13


def test_restated_psdscale_hermitian_block_against_direct_formula():
    rng = np.random.default_rng(5)
    n = 5
    K = cones.finish_K({"l": 1.0, "q": np.zeros(0), "s": np.array([float(n)]), "rsdpN": 0})
    U = np.triu(rng.standard_normal((n, n)) + 1j * rng.standard_normal((n, n)))
    X = rng.standard_normal((n, n)) + 1j * rng.standard_normal((n, n))
    X = X + X.conj().T
    u = np.r_[U.real.ravel(order="F"), U.imag.ravel(order="F")]
    x = np.r_[X.real.ravel(order="F"), X.imag.ravel(order="F")]
    y = restate.psdscale(u, x, K, True)
    Y = U.conj().T @ X @ U
    Yi = Y.imag.copy()
    Yi[np.diag_indices(n)] = 0.0
    assert relerr(y, np.r_[Y.real.ravel(order="F"), Yi.ravel(order="F")]) <= 1e-14
