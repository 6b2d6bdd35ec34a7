"""Parity of the CUDA invcholfac / getada1 / getada2 / getada3 / psdscale plugins against the
reference (oracle/_ref MEX for the C targets, oracle/restate.py for the M-only psdscale),
through the same mexFunction boundary.  Gates: ADA, absd, udsqr <= 1e-10 relative."""
import os
import sys

import numpy as np
import pytest
import scipy.sparse as sp

from helpers import ROOT, gpu, ref, relerr
from sedumi_b200.host import cones, problems, setup

sys.path.insert(0, os.path.join(ROOT, "oracle"))
import restate  # noqa: E402

pytestmark = pytest.mark.gpu


def _DAtq(S, d):
    """DAt.q as getDAtm builds it (getDAtm.m:40-43), via the reference ddot MEX."""
    K = S.K
    nq = len(K["q"])
    tr = setup.extractA(S.At, S.Ablkjc, 1, 2, int(K["mainblks"][0]), int(K["mainblks"][1]))
    if nq == 0:
        return tr
    Q = sp.diags(d["q1"]) @ tr + ref.ddot(d["q2"], S.At, K["qblkstart"].reshape(1, -1), S.Ablkjc)
    return sp.csc_matrix(Q)


def _chain(plug, S, d, udsqr):
    Km = S.Kmex()
    ADA0 = sp.csc_matrix((np.zeros(S.ADA.nnz), S.ADA.indices, S.ADA.indptr), shape=S.ADA.shape)
    A1 = plug.getada1(ADA0, S.At, S.Ablkjc[:, 2], S.Aord["lqperm"], {"l": d["l"], "det": d["det"]},
                      S.K["qblkstart"].reshape(1, -1))
    A2 = plug.getada2(A1, {"q": _DAtq(S, d)}, S.Aord, Km)
    A3, absd = plug.getada3(A2, S.At, S.Ablkjc[:, 2], S.Aord, udsqr, Km, nlhs=2)
    return A1, A2, A3, absd


def _problem(name):
    if name == "small_mixed":
        raw = problems.synth_small_mixed()
    elif name == "small_sdp":
        raw = problems.synth_small_mixed(seed=7, m=30, l=0, q=(), s=(9, 6), density=0.25)
    elif name == "small_free_rot":
        raw = problems.synth_small_mixed(seed=9, m=25, l=3, q=(3,), s=(5,), f=2, r=(4,))
    elif name == "maxcut_small":                      # A_j = e_j e_j': W only needed on the diagonal (sparse mode)
        raw = problems.synth_maxcut(n=48, p=0.2, seed=2)
    elif name == "blockdiag_sparse":                  # very sparse coefficients in larger blocks (sparse mode)
        raw = problems.synth_blockdiag_sdp(nblk=3, n=40, m=30, nlink=4, density=0.004, seed=6)
    elif name == "strip_even_optin":                  # different seeds: a plan of their own (the switch is read at plan build)
        raw = problems.synth_blockdiag_sdp(nblk=2, n=168, m=70, nlink=5, density=0.02, seed=22)
    elif name == "strip_odd_optin":
        raw = problems.synth_blockdiag_sdp(nblk=3, n=141, m=60, nlink=6, density=0.01, seed=23)
    elif name == "strip_mixed_optin":
        raw = problems.synth_small_mixed(seed=24, m=36, l=2, q=(3,), s=(130, 40), density=0.02)
    elif name == "strip_even":                        # blocks of order 97..208: (pair, column strip) work items (ada_strip.cuh)
        raw = problems.synth_blockdiag_sdp(nblk=2, n=168, m=70, nlink=5, density=0.02, seed=12)
    elif name == "strip_odd":                         # odd order: the scalar (unvectorised) staging paths
        raw = problems.synth_blockdiag_sdp(nblk=3, n=141, m=60, nlink=6, density=0.01, seed=13)
    elif name == "strip_mixed":                       # a large and a small block in every constraint, plus LP / Lorentz
        raw = problems.synth_small_mixed(seed=14, m=36, l=2, q=(3,), s=(130, 40), density=0.02)
    elif name == "blockdiag_small":
        raw = problems.synth_blockdiag_sdp(nblk=4, n=20, m=60, nlink=6, density=0.05, seed=5)
    else:
        raw = problems.load_fixture(name)
    At, b, c, K = cones.pretransfo(*raw)[:4]
    return setup.build_setup(At, b, c, K)


@pytest.mark.parametrize("name", ["small_mixed", "small_sdp", "small_free_rot", "blockdiag_small", "maxcut_small",
                                  "blockdiag_sparse", "arch0", "control07", "strip_even", "strip_odd", "strip_mixed"])
@pytest.mark.parametrize("kind", ["S0", "S1"])
def test_ada_chain(name, kind):
    S = _problem(name)
    d = setup.sdinit_scaling(S.b, S.c, S.K) if kind == "S0" else problems.scaling(S.K, "S1", seed=11)
    Km = S.Kmex()
    ur = ref.invcholfac(d["u"], Km, d["perm"])
    ug = gpu.invcholfac(d["u"], Km, d["perm"])
    assert relerr(ug, ur) <= 1e-10
    R = _chain(ref, S, d, ur)
    G = _chain(gpu, S, d, ur)
    for a, b_, nm in zip(G[:3], R[:3], ("getada1", "getada2", "getada3")):
        assert np.array_equal(a.indptr, b_.indptr) and np.array_equal(a.indices, b_.indices), nm
        assert relerr(a.data, b_.data) <= 1e-10, nm
    assert relerr(G[3], R[3]) <= 1e-10
    assert abs(G[2] - G[2].T).max() == 0.0            # spmakesym gives exact symmetry


@pytest.mark.parametrize("name", ["strip_even", "strip_odd", "strip_mixed"])
def test_ada_strip_path(name, monkeypatch):
    """The opt-in (pair, column strip) kernel of ada_strip.cuh (SB200_STRIP_ADA3=1, read when the plan is built)."""
    monkeypatch.setenv("SB200_STRIP_ADA3", "1")
    S = _problem(name + "_optin")
    d = problems.scaling(S.K, "S1", seed=21)
    ur = ref.invcholfac(d["u"], S.Kmex(), d["perm"])
    R, G = _chain(ref, S, d, ur), _chain(gpu, S, d, ur)
    assert relerr(G[2].data, R[2].data) <= 1e-10 and relerr(G[3], R[3]) <= 1e-10


def test_ada_late_scaling():
    S = _problem("small_sdp")
    d = problems.scaling(S.K, "S2", seed=5)
    ur = ref.invcholfac(d["u"], S.Kmex(), d["perm"])
    assert relerr(gpu.invcholfac(d["u"], S.Kmex(), d["perm"]), ur) <= 1e-10
    R, G = _chain(ref, S, d, ur), _chain(gpu, S, d, ur)
    assert relerr(G[2].data, R[2].data) <= 1e-10 and relerr(G[3], R[3]) <= 1e-10


@pytest.mark.parametrize("s", [(1,), (5,), (64,), (65, 3), (130, 70, 35)])
@pytest.mark.parametrize("transp", [0, 1])
@pytest.mark.parametrize("use_perm", [False, True])
def test_psdscale(s, transp, use_perm):
    K = cones.finish_K({"l": 1, "q": np.zeros(0), "s": np.array(s, dtype=float)})
    d = problems.scaling(K, "S1", seed=sum(s))
    if not use_perm:
        d["perm"] = np.zeros((0, 0))
    rng = np.random.default_rng(3)
    lenud = int(sum(n * n for n in s))
    x = rng.standard_normal(1 + lenud)                    # PSD part is the tail of x
    yr = restate.psdscale({"u": d["u"], "perm": d["perm"]}, x, K, transp)
    yg = gpu.psdscale({"u": d["u"], "perm": d["perm"]}, x, cones.K_for_mex(K), float(transp))
    assert relerr(yg.ravel(), yr) <= 1e-10
    # raw-vector form of ud (psdscale.m:71-74)
    yr2 = restate.psdscale(d["u"], x, K, transp)
    yg2 = gpu.psdscale(d["u"], x, cones.K_for_mex(K), float(transp))
    assert relerr(yg2.ravel(), yr2) <= 1e-10


def test_psdscale_roundtrip_property():
    """Size-independent property at a larger size: psdscale with T then with inv(T) is the identity."""
    n = 300
    K = cones.finish_K({"l": 1, "q": np.zeros(0), "s": np.array([float(n)])})
    rng = np.random.default_rng(1)
    U = np.triu(rng.standard_normal((n, n)) * 0.05 + np.eye(n))
    Ui = np.linalg.inv(U)
    X = rng.standard_normal((n, n)); X = X + X.T
    Km = cones.K_for_mex(K)
    Y = gpu.psdscale(U.ravel(order="F"), X.ravel(order="F"), Km, 1.0)
    X2 = gpu.psdscale(Ui.ravel(order="F"), Y.ravel(), Km, 1.0)
    assert relerr(X2.ravel(), X.ravel(order="F")) <= 1e-9


def test_invcholfac_empty_perm_and_identity():
    K = cones.finish_K({"l": 1, "q": np.zeros(0), "s": np.array([6.0, 4.0])})
    d = problems.scaling(K, "S1", seed=2)
    Km = cones.K_for_mex(K)
    assert relerr(gpu.invcholfac(d["u"], Km), ref.invcholfac(d["u"], Km)) <= 1e-12
    assert relerr(gpu.invcholfac(d["u"], Km, np.zeros((0, 0))), ref.invcholfac(d["u"], Km, np.zeros((0, 0)))) <= 1e-12


def test_getada2_empty_DAtq_returns_input():
    """K.q non-empty but DAt.q without nonzeros (every Lorentz cone dense, getDAtm.m:44): the reference returns
    mxDuplicateArray(ADA_IN) (getada2.c:150-153) -- the plugin must return the input VALUES, not scratch."""
    S = _problem("small_mixed")
    d = problems.scaling(S.K, "S1", seed=4)
    Km = S.Kmex()
    ADA0 = sp.csc_matrix((np.zeros(S.ADA.nnz), S.ADA.indices, S.ADA.indptr), shape=S.ADA.shape)
    A1 = ref.getada1(ADA0, S.At, S.Ablkjc[:, 2], S.Aord["lqperm"], {"l": d["l"], "det": d["det"]},
                     S.K["qblkstart"].reshape(1, -1))
    empty = {"q": sp.csc_matrix((len(S.K["q"]), S.m))}
    Ar = ref.getada2(A1, empty, S.Aord, Km)
    Ag = gpu.getada2(A1, empty, S.Aord, Km)
    assert np.array_equal(Ag.indptr, Ar.indptr) and np.array_equal(Ag.indices, Ar.indices)
    assert np.array_equal(Ag.data, Ar.data) and np.array_equal(Ag.data, A1.data)


def test_psdscale_sparse_x():
    """psdscale.m accepts a sparse x (it sparsifies blocks itself, psdscale.m:100-102); so does the plugin."""
    s = (7, 4)
    K = cones.finish_K({"l": 1, "q": np.zeros(0), "s": np.array(s, dtype=float)})
    d = problems.scaling(K, "S1", seed=11)
    rng = np.random.default_rng(5)
    lenud = int(sum(n * n for n in s))
    x = rng.standard_normal(1 + lenud) * (rng.random(1 + lenud) < 0.2)
    yr = restate.psdscale({"u": d["u"], "perm": d["perm"]}, x, K, 0)
    yg = gpu.psdscale({"u": d["u"], "perm": d["perm"]}, sp.csc_matrix(x.reshape(-1, 1)), cones.K_for_mex(K), 0.0)
    assert relerr(yg.ravel(), yr) <= 1e-10
