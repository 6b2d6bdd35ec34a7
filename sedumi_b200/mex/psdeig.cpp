// [lab,q] = psdeig(x,K)   spectral coefficients (and eigenvectors) of every PSD block (psdeig.m:40-96; M code in the
// reference, a MEX of the same name shadows it)
#include "mex_common.h"

void mexFunction(int nlhs, mxArray *plhs[], int nrhs, const mxArray *prhs[]) {
  MEX_REQUIRE(nrhs >= 2, "psdeig requires 2 input arguments.");
  MEX_REQUIRE(nlhs <= 2, "psdeig generates 2 output arguments.");
  ConeK K;
  read_cone(prhs[1], K);
  if (K.sdpN == 0) { plhs[0] = mxCreateDoubleMatrix(0, 0, mxREAL); if (nlhs >= 2) plhs[1] = mxCreateDoubleMatrix(0, 0, mxREAL); return; }
  MEX_REQUIRE(K.rsdpN == K.sdpN, "psdeig: Hermitian PSD blocks are not handled by the CUDA plugin");
  const sb_idx N = K.rDim;
  MEX_REQUIRE((sb_idx)numel(prhs[0]) >= N, "x size mismatch");
  MEX_REQUIRE(!mxIsSparse(prhs[0]), "x must be full");
  plhs[0] = mxCreateDoubleMatrix((mwSize)K.rLen, 1, mxREAL);
  if (nlhs >= 2) plhs[1] = mxCreateDoubleMatrix((mwSize)N, 1, mxREAL);
  int rc = sb200_psdeig(K.sdpN, K.s.data(), mxGetPr(prhs[0]) + (numel(prhs[0]) - (mwSize)N), mxGetPr(plhs[0]),
                        nlhs >= 2 ? mxGetPr(plhs[1]) : NULL);
  if (rc) {
    mxDestroyArray(plhs[0]); plhs[0] = NULL;
    if (nlhs >= 2) { mxDestroyArray(plhs[1]); plhs[1] = NULL; }
    sb_check(rc, "psdeig");
  }
}
