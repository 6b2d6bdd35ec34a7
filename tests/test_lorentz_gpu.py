"""Parity of the Lorentz stream plugins (ddot, qblkmul, quadadd) against the reference MEX.
quadadd is an error-free transformation: bit-exact.  ddot/qblkmul: 1e-12 relative."""
import numpy as np
import pytest
import scipy.sparse as sp

from helpers import gpu, ref, relerr, same
from sedumi_b200.host import cones, problems, setup

pytestmark = pytest.mark.gpu


def test_quadadd_bit_exact():
    rng = np.random.default_rng(0)
    n = 100003
    xhi = rng.standard_normal(n) * 10.0 ** rng.integers(-8, 8, n)
    xlo = xhi * 1e-17 * rng.standard_normal(n)
    y = rng.standard_normal(n) * 10.0 ** rng.integers(-8, 8, n)
    y[::7] = 0.0
    xhi[::11] = 0.0
    zr = ref.quadadd(xhi, xlo, y, nlhs=2)
    zg = gpu.quadadd(xhi, xlo, y, nlhs=2)
    assert same(zg[0], zr[0]) and same(zg[1], zr[1])


def test_quadadd_empty():
    z = gpu.quadadd(np.zeros((0, 1)), np.zeros((0, 1)), np.zeros((0, 1)), nlhs=2)
    assert z[0].size == 0 and z[1].size == 0


@pytest.mark.parametrize("q", [(3,), (3, 3, 3), (2, 7, 40, 3), tuple([3] * 793)])
def test_qblkmul_and_dense_ddot(q):
    K = cones.finish_K({"l": 5, "q": np.array(q, dtype=float), "s": np.zeros(0)})
    rng = np.random.default_rng(len(q))
    nq = len(q)
    qdim = int(sum(q)) - nq
    mu = rng.standard_normal(nq)
    dvec = rng.standard_normal(qdim)
    bs = K["qblkstart"].reshape(1, -1)
    assert relerr(gpu.qblkmul(mu, dvec, bs), ref.qblkmul(mu, dvec, bs)) <= 1e-14
    # full-length x (LP + Lorentz): d and x point into the norm-bound part (qblkmul.c:88-97, ddot.c:213-233)
    xfull = rng.standard_normal(int(K["N"]))
    assert relerr(gpu.qblkmul(mu, xfull, bs), ref.qblkmul(mu, xfull, bs)) <= 1e-14
    X = rng.standard_normal((int(K["N"]), 3))
    assert relerr(gpu.ddot(dvec, X, bs), ref.ddot(dvec, X, bs)) <= 1e-12
    Xq = rng.standard_normal((nq + qdim, 2))             # [traces; norm-bound] layout
    assert relerr(gpu.ddot(dvec, Xq, bs), ref.ddot(dvec, Xq, bs)) <= 1e-12


@pytest.mark.parametrize("name", ["nb", "small_mixed"])
def test_sparse_ddot_on_At(name):
    """The getDAtm call: ddot(d.q2, A, K.qblkstart, Ablkjc) (getDAtm.m:43)."""
    raw = problems.load_fixture("nb") if name == "nb" else problems.synth_small_mixed()
    At, b, c, K = cones.pretransfo(*raw)[:4]
    S = setup.build_setup(At, b, c, K)
    d = problems.scaling(K, "S1", seed=4)
    bs = K["qblkstart"].reshape(1, -1)
    yr = ref.ddot(d["q2"], S.At, bs, S.Ablkjc)
    yg = gpu.ddot(d["q2"], S.At, bs, S.Ablkjc)
    assert yr.shape == yg.shape
    assert np.array_equal(yr.indptr, yg.indptr) and np.array_equal(yr.indices, yg.indices)
    assert relerr(yg.data, yr.data) <= 1e-12
