// [LL,Ld,Lskip,Ladd] = blkchol(L,X[,pars[,absd]])  -- CUDA plugin, same contract as the
// reference MEX (blkchol.c:58-69 signature, :239-440 mexFunction).
#include "mex_common.h"

void mexFunction(int nlhs, mxArray *plhs[], int nrhs, const mxArray *prhs[]) {
  MEX_REQUIRE(nrhs >= 2, "blkchol requires more input arguments");
  MEX_REQUIRE(nlhs <= 4, "blkchol produces less output arguments");
  const mxArray *L_IN = prhs[0], *P_IN = prhs[1];
  mwSize m = mxGetM(P_IN);
  MEX_REQUIRE(m == mxGetN(P_IN), "P must be square");
  MEX_REQUIRE(mxIsSparse(P_IN), "P must be sparse");
  MEX_REQUIRE(mxIsStruct(L_IN), "Parameter `L' should be a structure.");
  const mxArray *Lperm = need_field(L_IN, "perm", "Missing field L.perm.");
  MEX_REQUIRE(numel(Lperm) == m, "perm size mismatch");
  const mxArray *LL = need_field(L_IN, "L", "Missing field L.L.");
  MEX_REQUIRE(mxGetM(LL) == m && mxGetN(LL) == m, "Size L.L mismatch.");
  MEX_REQUIRE(mxIsSparse(LL), "L.L should be sparse.");
  const mxArray *Lxs = need_field(L_IN, "xsuper", "Missing field L.xsuper.");
  MEX_REQUIRE(numel(Lxs) >= 1 && numel(Lxs) - 1 <= m, "Size L.xsuper mismatch.");
  need_field(L_IN, "tmpsiz", "Missing field L.tmpsiz.");     // workspace hint of the CPU code: unused here
  sb200_chol_pars pars = {1E-20, 1E-12, 5E2};                 // defaults of blkchol.c:292-294
  const double *absd = NULL;
  if (nrhs >= 3) {
    const mxArray *PARS = prhs[2], *f;
    MEX_REQUIRE(mxIsStruct(PARS), "Parameter `pars' should be a structure.");
    if ((f = mxGetField(PARS, 0, "canceltol")) != NULL) pars.canceltol = mxGetScalar(f);
    if ((f = mxGetField(PARS, 0, "maxu")) != NULL) pars.maxu = mxGetScalar(f);
    if ((f = mxGetField(PARS, 0, "abstol")) != NULL) { pars.abstol = mxGetScalar(f); if (pars.abstol < 0.0) pars.abstol = 0.0; }
    if ((f = mxGetField(PARS, 0, "delay")) != NULL && mxGetScalar(f) != 0.0)
      mexErrMsgTxt("blkchol: pars.delay is not supported by the CUDA plugin (sedumi.m never sets it).");
    if (nrhs >= 4) {
      MEX_REQUIRE(numel(prhs[3]) == m, "absd size mismatch");
      absd = mxGetPr(prhs[3]);
    }
  }
  std::vector<sb_idx> perm, xsuper;
  idx_from_double(Lperm, perm, 1, "L.perm");
  idx_from_double(Lxs, xsuper, 1, "L.xsuper");
  const mwIndex *Ljc = mxGetJc(LL), *Lir = mxGetIr(LL);
  mwSize nnzL = Ljc[m];
  mxArray *myplhs[4];
  myplhs[0] = sparse_with_pattern(m, m, Ljc, Lir);
  myplhs[1] = mxCreateDoubleMatrix(m, 1, mxREAL);
  std::vector<sb_idx> skip(m ? m : 1), add(m ? m : 1);
  std::vector<double> skipv(m ? m : 1), addv(m ? m : 1);
  sb_idx nskip = 0, nadd = 0;
  int rc = sb200_blkchol((sb_idx)m, (sb_idx)xsuper.size() - 1, xsuper.data(), as_idx(Ljc), as_idx(Lir), perm.data(),
                         as_idx(mxGetJc(P_IN)), as_idx(mxGetIr(P_IN)), mxGetPr(P_IN), absd, pars,
                         mxGetPr(myplhs[0]), mxGetPr(myplhs[1]), skip.data(), skipv.data(), &nskip,
                         add.data(), addv.data(), &nadd);
  if (rc) { mxDestroyArray(myplhs[0]); mxDestroyArray(myplhs[1]); sb_check(rc, "blkchol"); }
  for (int o = 2; o < 4; o++) {
    sb_idx n = (o == 2) ? nskip : nadd;
    const sb_idx *ix = (o == 2) ? skip.data() : add.data();
    const double *vx = (o == 2) ? skipv.data() : addv.data();
    myplhs[o] = mxCreateSparse(m, 1, n > 0 ? (mwSize)n : 1, mxREAL);
    mwIndex *ir = mxGetIr(myplhs[o]), *jc = mxGetJc(myplhs[o]);
    double *pr = mxGetPr(myplhs[o]);
    for (sb_idx i = 0; i < n; i++) { ir[i] = (mwIndex)ix[i]; pr[i] = vx[i]; }
    jc[0] = 0; jc[1] = (mwIndex)n;
  }
  int nout = nlhs > 1 ? nlhs : 1;
  for (int i = 0; i < 4; i++) {
    if (i < nout) plhs[i] = myplhs[i];
    else mxDestroyArray(myplhs[i]);
  }
}
