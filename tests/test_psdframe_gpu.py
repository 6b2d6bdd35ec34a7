"""Parity of psdframeit / psdinvjmul / urotorder / givensrot plugins against the reference MEX.
Frames (Householder product form) come from the reference's own qrK, as in updtransfo.m:107."""
import numpy as np
import pytest

from helpers import gpu, ref, relerr
from sedumi_b200.host import cones, problems

pytestmark = pytest.mark.gpu


def _K(s):
    return cones.finish_K({"l": 2.0, "q": np.array([3.0]), "s": np.array(s, dtype=float)})


def _frames(K, seed, qr=ref):
    rng = np.random.default_rng(seed)
    blocks = [rng.standard_normal((int(n), int(n))) for n in K["s"]]
    x = np.concatenate([b.ravel(order="F") for b in blocks])
    return qr.qrK(x, cones.K_for_mex(K))             # vfrm.s layout: reflectors + beta column


@pytest.mark.parametrize("s", [(1,), (2,), (7,), (33, 5), (70, 35), (130,), (200, 40), (257,), (129, 2, 161)])
def test_psdframeit(s):
    K = _K(s)
    Km = cones.K_for_mex(K)
    frms = _frames(K, sum(s))
    rng = np.random.default_rng(1)
    lab = rng.uniform(0.1, 3.0, int(sum(s)))
    xr = ref.psdframeit(lab, frms, Km)
    xg = gpu.psdframeit(lab, frms, Km)
    assert relerr(xg, xr) <= 1e-10
    # full-length lab (LP + 2*|K.q| + PSD): psdframeit.c:131-134
    labfull = np.r_[rng.standard_normal(int(K["l"]) + 2), lab]
    assert relerr(gpu.psdframeit(labfull, frms, Km), xr) <= 1e-10


@pytest.mark.parametrize("s", [(1,), (6,), (40, 9), (70, 35), (100,), (150, 20)])
def test_psdinvjmul(s):
    K = _K(s)
    Km = cones.K_for_mex(K)
    frms = _frames(K, 5 + sum(s))
    rng = np.random.default_rng(2)
    xlab = rng.uniform(0.5, 2.0, int(sum(s)))
    ys = []
    for n in s:
        Y = rng.standard_normal((n, n)); ys.append((Y + Y.T).ravel(order="F"))
    y = np.concatenate(ys)
    zr = ref.psdinvjmul(xlab, frms, y, Km)
    zg = gpu.psdinvjmul(xlab, frms, y, Km)
    assert relerr(zg, zr) <= 1e-10
    # defining property: X Z + Z X = 2 Y with X = psdframeit(xlab, frms)
    X = gpu.psdframeit(xlab, frms, Km).ravel()
    off = 0
    for n in s:
        Xk = X[off:off + n * n].reshape(n, n, order="F"); Zk = zg.ravel()[off:off + n * n].reshape(n, n, order="F")
        Yk = y[off:off + n * n].reshape(n, n, order="F")
        assert np.abs(Xk @ Zk + Zk @ Xk - 2 * Yk).max() <= 1e-9 * max(1.0, np.abs(Yk).max())
        off += n * n


def _bad_factor(n, rng, scale):
    """Upper-triangular U whose leading columns are tiny: forces pivoting in rotorder."""
    U = np.triu(rng.standard_normal((n, n)))
    U[np.diag_indices(n)] = np.abs(U[np.diag_indices(n)]) + 0.5
    U = U * scale[None, :]
    return U + np.triu(U, 1).T


@pytest.mark.parametrize("s,maxu", [((1,), 1.1), ((6,), 1.1), ((20, 7), 1.1), ((70, 35), 1.1), ((50,), 3.0)])
def test_urotorder_and_givensrot_bit_exact(s, maxu):
    K = _K(s)
    Km = cones.K_for_mex(K)
    rng = np.random.default_rng(sum(s))
    us = []
    for n in s:
        scale = 10.0 ** rng.uniform(-3, 0, n)
        scale[: max(n // 3, 1)] *= 1e-3
        us.append(_bad_factor(n, rng, scale).ravel(order="F"))
    u = np.concatenate(us)
    permin = np.concatenate([rng.permutation(n) + 1.0 for n in s])
    R = ref.urotorder(u, Km, maxu, permin, nlhs=4)
    G = gpu.urotorder(u, Km, maxu, permin, nlhs=4)
    assert np.array_equal(R[1], G[1]), "perm"
    assert np.array_equal(R[2], G[2]), "gjc"
    assert R[3].shape == G[3].shape and np.array_equal(R[3], G[3]), "g"
    assert np.array_equal(R[0], G[0]), "u"
    if len(s) > 1 or s[0] > 1:
        assert R[2].max() > 0                       # rotations were actually needed
    # without permIN
    R2 = ref.urotorder(u, Km, maxu, nlhs=2)
    G2 = gpu.urotorder(u, Km, maxu, nlhs=2)
    assert np.array_equal(R2[1], G2[1]) and np.array_equal(R2[0], G2[0])
    # givensrot with that rotation list on a random Q
    x = rng.standard_normal(u.size)
    yr = ref.givensrot(R[2], R[3], x, Km)
    yg = gpu.givensrot(R[2], R[3], x, Km)
    assert np.array_equal(yr, yg)


def test_urotorder_no_rotation_needed():
    K = _K((12,))
    Km = cones.K_for_mex(K)
    u = np.eye(12).ravel()
    R = ref.urotorder(u, Km, 1.1, nlhs=4)
    G = gpu.urotorder(u, Km, 1.1, nlhs=4)
    assert R[3].size == 0 and G[3].size == 0 and np.array_equal(R[1], G[1]) and np.array_equal(R[0], G[0])
    x = np.arange(144.0)
    assert np.array_equal(gpu.givensrot(G[2], G[3], x, Km), ref.givensrot(R[2], R[3], x, Km))


def test_psdframeit_gemm_wy_path_wide_panels(monkeypatch):
    """Blocks beyond ~2300 accumulate Q through the tile-GEMM engine with 128-reflector panels (compact WY).  The
    path is forced at a size the reference handles quickly (the plan cache is keyed by the block sizes: 301 and 143
    appear nowhere else in the suite).  The frames come from the CUDA qrK (checked against the reference's in
    tests/test_psdalg_gpu.py) and go to both sides, so that the reference's answers for this test stay small enough to
    store."""
    monkeypatch.setenv("SB200_WY_GEMM_MIN_N", "100")
    s = (301, 143)
    K = _K(s)
    Km = cones.K_for_mex(K)
    frms = _frames(K, 77, qr=gpu)
    rng = np.random.default_rng(3)
    lab = rng.uniform(0.1, 3.0, int(sum(s)))
    assert relerr(gpu.psdframeit(lab, frms, Km), ref.psdframeit(lab, frms, Km)) <= 1e-10
    ys = []
    for n in s:
        Y = rng.standard_normal((n, n)); ys.append((Y + Y.T).ravel(order="F"))
    y = np.concatenate(ys)
    assert relerr(gpu.psdinvjmul(lab, frms, y, Km), ref.psdinvjmul(lab, frms, y, Km)) <= 1e-10
