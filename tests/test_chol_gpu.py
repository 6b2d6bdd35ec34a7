"""Parity of the CUDA blkchol / fwblkslv / bwblkslv plugins against the reference MEX
(oracle/_ref), called through the same mexFunction boundary on the same inputs.
Gates (SURVEY.md section 8d): L, d <= 1e-10 relative; identical skip/add index sets."""
import numpy as np
import pytest
import scipy.sparse as sp

from helpers import CHOL_PARS, check_chol, dense_L, full_pattern, gpu, random_sparse_spd, random_spd, ref, relerr
from sedumi_b200.host import symbolic

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("m", [1, 2, 7, 33, 128, 129, 161, 300, 666])
def test_dense_single_supernode(m):
    X = random_spd(m, seed=m, cond=1e4)
    check_chol(dense_L(m), full_pattern(X), CHOL_PARS, np.diag(X).copy())


def test_dense_no_absd_default_pars():
    m = 90
    X = random_spd(m, seed=5, cond=1e3)
    LLr, dr = ref.blkchol(dense_L(m), full_pattern(X), nlhs=2)
    LLg, dg = gpu.blkchol(dense_L(m), full_pattern(X), nlhs=2)
    assert relerr(LLg.data, LLr.data) <= 1e-10 and relerr(dg, dr) <= 1e-10


@pytest.mark.parametrize("m,rank", [(40, 30), (150, 100), (260, 200)])
def test_rank_deficient_skips(m, rank):
    """Dependent constraints: pivots collapse below canceltol*absd and must be skipped
    exactly where the reference skips them (blkchol2.c:157-161)."""
    rng = np.random.default_rng(m)
    B = rng.standard_normal((m, rank))
    X = B @ B.T
    absd = np.einsum("ij,ij->i", np.abs(B), np.abs(B))
    pars = dict(CHOL_PARS, canceltol=1e-9)
    (LLr, dr, skr, adr), _ = check_chol(dense_L(m), full_pattern(X), pars, absd, tol=1e-7)
    assert skr.nnz >= m - rank - 2


@pytest.mark.parametrize("m,maxu", [(60, 5e2), (200, 5e2), (300, 50.0)])
def test_diag_add_path(m, maxu):
    """Badly scaled matrix + small maxu: the stability test (x_kk < ub) fires and pivots get
    raised ("add").  Exercises the reference's idamax-indexed threshold (blkchol2.c:66-70,122)."""
    rng = np.random.default_rng(1000 + m)
    s = 10.0 ** rng.uniform(-5, 5, m)
    X = random_spd(m, seed=m + 3, cond=1e2) * np.outer(s, s)
    pars = dict(CHOL_PARS, maxu=maxu)
    (LLr, dr, skr, adr), _ = check_chol(dense_L(m), full_pattern(X), pars, np.diag(X).copy(), tol=1e-8)
    assert adr.nnz > 0


@pytest.mark.parametrize("m,density,seed", [(60, 0.05, 1), (300, 0.01, 2), (800, 0.004, 3), (500, 0.02, 4)])
def test_sparse_multisupernode(m, density, seed):
    X = random_sparse_spd(m, density, seed)
    L = symbolic.symbolic_factor(X)
    assert len(L["xsuper"]) - 1 > 1
    check_chol(L, X, CHOL_PARS, np.asarray(X.diagonal()).copy())


def test_sparse_reference_symbolic():
    """Same, with the reference's own ordering + symbolic factorisation as the producer of L."""
    X = random_sparse_spd(400, 0.01, 7)
    perm = ref.ordmmdmex(X)
    L = ref.symfctmex(X, perm)
    L["tmpsiz"] = ref.choltmpsiz(L)
    check_chol(L, X, CHOL_PARS, np.asarray(X.diagonal()).copy())


def test_arrow_structure():
    """Block-arrow ADA (config 4 shape, small): independent subtrees + a dense border."""
    rng = np.random.default_rng(11)
    nb, bs, border = 6, 40, 150
    m = nb * bs + border
    blocks = [random_spd(bs, seed=k, cond=1e2) + bs * np.eye(bs) for k in range(nb)]
    X = sp.lil_matrix((m, m))
    for k, Bk in enumerate(blocks):
        X[k * bs:(k + 1) * bs, k * bs:(k + 1) * bs] = Bk
    C = 0.1 * rng.standard_normal((border, nb * bs))
    X[nb * bs:, :nb * bs] = C
    X[:nb * bs, nb * bs:] = C.T
    X[nb * bs:, nb * bs:] = random_spd(border, seed=99, cond=1e2) + border * np.eye(border)
    X = sp.csc_matrix(X)
    L = symbolic.symbolic_factor(X, perm=np.arange(m))
    check_chol(L, X, CHOL_PARS, np.asarray(X.diagonal()).copy())


@pytest.mark.parametrize("m,nrhs", [(1, 1), (50, 1), (300, 3), (666, 1)])
def test_solves_dense(m, nrhs):
    """Both solves on the same factor; it comes from the CUDA blkchol (checked against the reference above), so that
    the reference's answers for this test stay small enough to store."""
    X = random_spd(m, seed=m + 17, cond=1e3)
    L = dense_L(m)
    LL, d = gpu.blkchol(L, full_pattern(X), CHOL_PARS, np.diag(X).copy(), nlhs=2)
    Lf = dict(L, L=LL)
    b = np.random.default_rng(m).standard_normal((m, nrhs))
    yr, yg = ref.fwblkslv(Lf, b), gpu.fwblkslv(Lf, b)
    assert relerr(yg, yr) <= 1e-10
    zr, zg = ref.bwblkslv(Lf, b), gpu.bwblkslv(Lf, b)
    assert relerr(zg, zr) <= 1e-10


@pytest.mark.parametrize("m,density,seed", [(300, 0.01, 2), (800, 0.004, 3)])
def test_solves_sparse_structure(m, density, seed):
    X = random_sparse_spd(m, density, seed)
    L = symbolic.symbolic_factor(X)
    LL, d = ref.blkchol(L, X, CHOL_PARS, np.asarray(X.diagonal()).copy(), nlhs=2)
    Lf = dict(L, L=LL)
    b = np.random.default_rng(seed).standard_normal((m, 2))
    assert relerr(gpu.fwblkslv(Lf, b), ref.fwblkslv(Lf, b)) <= 1e-10
    assert relerr(gpu.bwblkslv(Lf, b), ref.bwblkslv(Lf, b)) <= 1e-10


def test_fwblkslv_sparse_rhs():
    m = 300
    X = random_sparse_spd(m, 0.01, 5)
    L = symbolic.symbolic_factor(X)
    LL, d = ref.blkchol(L, X, CHOL_PARS, np.asarray(X.diagonal()).copy(), nlhs=2)
    Lf = dict(L, L=LL)
    B = sp.random(m, 4, density=0.02, random_state=np.random.RandomState(3), format="csc")
    ysymb = ref.symbfwblk(Lf, B)
    yr = ref.fwblkslv(Lf, B, ysymb)
    yg = gpu.fwblkslv(Lf, B, ysymb)
    assert np.array_equal(yr.indices, yg.indices)
    assert relerr(yg.data, yr.data) <= 1e-10


def test_solution_through_factor_and_solves():
    """End of the chain: x = ADA \\ r via our factor + our solves, vs numpy."""
    m = 200
    X = random_spd(m, seed=3, cond=1e4)
    L = dense_L(m)
    LL, d = gpu.blkchol(L, full_pattern(X), CHOL_PARS, np.diag(X).copy(), nlhs=2)
    Lf = dict(L, L=LL)
    r = np.random.default_rng(0).standard_normal((m, 1))
    y = gpu.bwblkslv(Lf, gpu.fwblkslv(Lf, r) / d)
    assert relerr(y, np.linalg.solve(X, r)) <= 1e-8
