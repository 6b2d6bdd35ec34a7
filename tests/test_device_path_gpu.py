"""The device-resident pipeline (sedumi_b200.device.HotPath, what bench.py's `value` times) against
the reference call sequence (oracle/refpath.py).  Gates: ADA/absd/factor 1e-10, search direction 1e-8."""
import os
import sys

import numpy as np
import pytest

from helpers import ROOT, relerr, same
from sedumi_b200.host import cones, problems, setup

sys.path.insert(0, os.path.join(ROOT, "oracle"))

pytestmark = pytest.mark.gpu


def _run(raw, perm=None, seed=3):
    import torch
    import refpath
    from sedumi_b200 import device
    At, b, c, K = cones.pretransfo(*raw)[:4]
    S = setup.build_setup(At, b, c, K, perm=perm)
    d = problems.scaling(K, "S1", seed=seed)
    rng = np.random.default_rng(seed)
    rhs = rng.standard_normal((S.m, 2))
    psd_x = rng.standard_normal(int((np.asarray(K["s"]) ** 2).sum()))
    lab, frms = problems.synth_frames(K["s"], seed=seed)
    hp = device.HotPath(S)
    st = hp.stream()
    with torch.cuda.stream(st):
        hp.set_scaling(d)
        hp.set_rhs(rhs)
        hp.psd_x[:psd_x.size].copy_(torch.from_numpy(psd_x))
        hp.set_frames(lab, frms)
        st.synchronize()
        hp.iteration(1, 2)
        hp.sync()
        n2 = psd_x.size
        tail = dict(z=hp.psd_z.cpu().numpy()[:n2].copy(), frame=hp.psd_f.cpu().numpy()[:n2],
                    u=hp.u_new.cpu().numpy()[:n2], perm=hp.perm_new.cpu().numpy()[:hp.sumn], gjc=hp.gjc.cpu().numpy()[:hp.sumn])
        out = dict(ADA=hp.ADA.cpu().numpy()[:S.ADA.nnz], absd=hp.absd.cpu().numpy()[:S.m],
                   d=hp.dvec.cpu().numpy()[:S.m], y=hp.y.cpu().numpy().T, psd=hp.psd_y.cpu().numpy()[:psd_x.size],
                   udsqr=hp.udsqr.cpu().numpy()[:psd_x.size])
    ref = refpath.RefHotPath(S).iteration(d, rhs, psd_x, 1, 2, frames=(lab, frms))
    if psd_x.size:
        # scaling-update tail: psdinvjmul, psdframeit, urotorder (discrete outputs exact), givensrot.
        # hp.psd_z was overwritten by givensrot (last call of the recipe), so z is checked separately below.
        rt = ref["tail"]
        assert relerr(tail["frame"], rt["frame"].ravel()) <= 1e-10
        assert same(tail["u"], rt["u"])
        assert np.array_equal(tail["perm"] + 1, rt["perm"].ravel().astype(np.int64))      # 1-based inside each block
        assert np.array_equal(tail["gjc"], rt["gjc"].ravel().astype(np.int64))
        assert relerr(tail["z"], rt["q"].ravel()) <= 1e-10
        with torch.cuda.stream(st):
            hp.psdinvjmul()
            hp.sync()
            assert relerr(hp.psd_z.cpu().numpy()[:psd_x.size], rt["z"].ravel()) <= 1e-9
    assert relerr(out["udsqr"], ref["udsqr"].ravel()) <= 1e-10
    assert relerr(out["ADA"], ref["ADA"].data) <= 1e-10
    assert relerr(out["absd"], ref["absd"].ravel()) <= 1e-10
    assert relerr(out["d"], ref["L"]["d"]) <= 1e-10
    assert relerr(out["y"], ref["y"]) <= 1e-8
    assert relerr(out["psd"], ref["psd"]) <= 1e-10
    return S


def test_control07():
    _run(problems.load_fixture("control07"))


def test_arch0():
    _run(problems.load_fixture("arch0"))


def test_nb_lorentz_only_device_path():
    """BASELINE config 2 (nb.mat: 793 Lorentz cones, no PSD block): getDAtm + getada1 + getada2 on the
    device against getada.m restated (the M path sedumi.m:446-448 takes), then factor/solve and the
    qblkmul/ddot/quadadd streams against the reference MEX."""
    import torch
    import refpath
    from sedumi_b200 import device
    At, b, c, K = cones.pretransfo(*problems.load_fixture("nb"))[:4]
    S = setup.build_setup(At, b, c, K)
    d = problems.scaling(K, "S1", seed=3)
    rng = np.random.default_rng(4)
    rhs = rng.standard_normal((S.m, 1))
    nq, qd = len(K["q"]), int((np.asarray(K["q"]) - 1).sum())
    mu, xq = rng.standard_normal(nq), rng.standard_normal(qd)
    rhi, rlo, ry = rng.standard_normal(S.m), 1e-17 * rng.standard_normal(S.m), rng.standard_normal(S.m)
    hp = device.HotPath(S)
    st = hp.stream()
    R = refpath.RefHotPath(S)
    with torch.cuda.stream(st):
        hp.set_scaling(d)
        hp.set_rhs(rhs)
        for dst, src in ((hp.q_mu, mu), (hp.q_x, xq), (hp.r_hi, rhi), (hp.r_lo, rlo), (hp.r_y, ry)):
            dst[:src.size].copy_(torch.from_numpy(src))
        st.synchronize()
        hp.iteration(1, 0)
        hp.sync()
        # DAt.q values (pattern order = CSC of the reference's DAt.q)
        import ctypes as C
        Q = R.DAtq(d)
        Q.sort_indices()
        nnz = hp.datq[3]
        assert nnz == Q.nnz
        got = np.empty(nnz)
        device.check(device.lib().sb200_d2h(got.ctypes.data_as(C.c_void_p), hp.datq[2], C.c_int64(8 * nnz)), "d2h")
        assert relerr(got, Q.data) <= 1e-12
        ref = R.iteration(d, rhs, np.zeros(0), 1, 0)
        assert relerr(hp.ADA.cpu().numpy()[:S.ADA.nnz], ref["ADA"].data) <= 1e-10
        assert relerr(hp.absd.cpu().numpy()[:S.m], ref["absd"].ravel()) <= 1e-10
        assert relerr(hp.dvec.cpu().numpy()[:S.m], ref["L"]["d"]) <= 1e-10
        assert relerr(hp.y.cpu().numpy().T, ref["y"]) <= 1e-8
        ls = R.lorentz_streams(d, mu, xq, rhi, rlo, ry)
        assert relerr(hp.q_y.cpu().numpy()[:qd], ls["y"].ravel()) <= 1e-14
        assert relerr(hp.q_dd.cpu().numpy()[:nq], ls["dd"].ravel()) <= 1e-12
        assert np.array_equal(hp.r_hi.cpu().numpy()[:S.m], ls["zhi"].ravel())
        assert np.array_equal(hp.r_lo.cpu().numpy()[:S.m], ls["zlo"].ravel())


def test_late_scaling_with_rotations():
    """S2 ("late") scaling: ill-conditioned factors, urotorder really pivots."""
    import refpath
    raw = problems.synth_small_mixed(seed=11, m=30, l=0, q=(), s=(12, 8), density=0.25)
    At, b, c, K = cones.pretransfo(*raw)[:4]
    d = problems.scaling(K, "S2", seed=5)
    Km = cones.K_for_mex(K)
    u, perm, gjc, g = refpath.ref_dir().urotorder(d["u"], Km, 1.1, nlhs=4)
    import torch
    from sedumi_b200 import device
    S = setup.build_setup(At, b, c, K)
    hp = device.HotPath(S)
    with torch.cuda.stream(hp.stream()):
        hp.set_scaling(d)
        lab, frms = problems.synth_frames(K["s"], seed=2)
        hp.set_frames(lab, frms)
        hp.psdframeit()
        hp.urotorder()
        hp.givensrot()
        hp.sync()
        assert same(hp.u_new.cpu().numpy()[:u.size], u)
        assert np.array_equal(hp.gjc.cpu().numpy()[:hp.sumn], gjc.ravel().astype(np.int64))
        assert np.array_equal(hp.perm_new.cpu().numpy()[:hp.sumn] + 1, perm.ravel().astype(np.int64))
        f = refpath.ref_dir().psdframeit(lab, frms, Km)
        q = refpath.ref_dir().givensrot(gjc, g, f, Km)
        assert relerr(hp.psd_z.cpu().numpy()[:u.size], q.ravel()) <= 1e-10
    assert gjc.ravel()[-1] > 0 or gjc.ravel()[11] > 0, "test input does not rotate; pick another seed"


def test_small_sdp():
    _run(problems.synth_small_mixed(seed=7, m=30, l=0, q=(), s=(9, 6), density=0.25))


def test_blockdiag_arrow_multisupernode():
    raw = problems.synth_blockdiag_sdp(nblk=6, n=30, m=200, nlink=20, density=0.04, seed=8)
    m = raw[0].shape[1]
    S = _run(raw, perm=np.arange(m))
    assert len(S.L["xsuper"]) - 1 > 1
