// [ux,ispos] = psdfactor(x,K)   Cholesky factor of every PSD block with a positive-definiteness flag (psdfactor.m:37-82)
#include "mex_common.h"

void mexFunction(int nlhs, mxArray *plhs[], int nrhs, const mxArray *prhs[]) {
  MEX_REQUIRE(nrhs >= 2, "psdfactor requires 2 input arguments.");
  MEX_REQUIRE(nlhs <= 2, "psdfactor generates 2 output arguments.");
  ConeK K;
  read_cone(prhs[1], K);
  MEX_REQUIRE(K.rsdpN == K.sdpN, "psdfactor: Hermitian PSD blocks are not handled by the CUDA plugin");
  const sb_idx N = K.rDim;
  MEX_REQUIRE((sb_idx)numel(prhs[0]) >= N, "x size mismatch");
  plhs[0] = mxCreateDoubleMatrix((mwSize)N, 1, mxREAL);
  int ispos = 1;
  int rc = sb200_psdfactor(K.sdpN, K.s.data(), mxGetPr(prhs[0]) + (numel(prhs[0]) - (mwSize)N), mxGetPr(plhs[0]), &ispos);
  if (rc) { mxDestroyArray(plhs[0]); plhs[0] = NULL; sb_check(rc, "psdfactor"); }
  if (nlhs >= 2) { plhs[1] = mxCreateDoubleMatrix(1, 1, mxREAL); mxGetPr(plhs[1])[0] = ispos ? 1.0 : 0.0; }
}
