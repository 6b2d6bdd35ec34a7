// y = bwblkslv(L,b)   y(L.perm,:) = L.L' \ b   (bwblkslv.c:48-54 signature, :182-298)
#include "mex_common.h"

void mexFunction(int nlhs, mxArray *plhs[], int nrhs, const mxArray *prhs[]) {
  MEX_REQUIRE(nrhs >= 2, "bwblkslv requires more input arguments.");
  MEX_REQUIRE(nlhs <= 1, "bwblkslv generates only 1 output argument.");
  const mxArray *L_IN = prhs[0];
  MEX_REQUIRE(mxIsStruct(L_IN), "Parameter `L' should be a structure.");
  const mxArray *f = need_field(L_IN, "perm", "Missing field L.perm.");
  mwSize m = numel(f);
  std::vector<sb_idx> perm, xsuper;
  idx_from_double(f, perm, 1, "L.perm");
  const mxArray *LL = need_field(L_IN, "L", "Missing field L.L.");
  MEX_REQUIRE(mxGetM(LL) == m && mxGetN(LL) == m, "Size L.L mismatch.");
  MEX_REQUIRE(mxIsSparse(LL), "L.L should be sparse.");
  f = need_field(L_IN, "xsuper", "Missing field L.xsuper.");
  MEX_REQUIRE(numel(f) >= 1 && numel(f) - 1 <= m, "Size L.xsuper mismatch.");
  idx_from_double(f, xsuper, 1, "L.xsuper");
  const mxArray *B = prhs[1];
  MEX_REQUIRE(mxGetM(B) == m, "Size mismatch b.");
  if (mxIsSparse(B))
    mexErrMsgTxt("bwblkslv: sparse right-hand sides are not supported by the CUDA plugin "
                 "(SeDuMi only calls bwblkslv with full b, sparbwslv.m:48).");
  mwSize n = mxGetN(B);
  plhs[0] = mxCreateDoubleMatrix(m, n, mxREAL);
  int rc = sb200_bwblkslv((sb_idx)m, (sb_idx)xsuper.size() - 1, xsuper.data(), as_idx(mxGetJc(LL)), as_idx(mxGetIr(LL)),
                          mxGetPr(LL), perm.data(), mxGetPr(B), mxGetPr(plhs[0]), (sb_idx)n);
  if (rc) { mxDestroyArray(plhs[0]); plhs[0] = NULL; sb_check(rc, "bwblkslv"); }
}
