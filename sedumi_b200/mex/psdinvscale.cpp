// y = psdinvscale(ud,x,K)   Y_k = T \ (X_k / T'), T = triu(U_k)   (psdinvscale.m:37-83)
#include "mex_common.h"

void mexFunction(int nlhs, mxArray *plhs[], int nrhs, const mxArray *prhs[]) {
  MEX_REQUIRE(nrhs >= 3, "psdinvscale requires 3 input arguments.");
  MEX_REQUIRE(nlhs <= 1, "psdinvscale generates 1 output argument.");
  ConeK K;
  read_cone(prhs[2], K);
  if (K.sdpN == 0) { plhs[0] = mxCreateDoubleMatrix(0, 0, mxREAL); return; }
  MEX_REQUIRE(K.rsdpN == K.sdpN, "psdinvscale: Hermitian PSD blocks are not handled by the CUDA plugin");
  const sb_idx N = K.rDim;
  MEX_REQUIRE((sb_idx)numel(prhs[0]) >= N, "ud size mismatch");
  MEX_REQUIRE((sb_idx)numel(prhs[1]) >= N && !mxIsSparse(prhs[1]), "x size mismatch");
  plhs[0] = mxCreateDoubleMatrix((mwSize)N, 1, mxREAL);
  int rc = sb200_psdinvscale(K.sdpN, K.s.data(), mxGetPr(prhs[0]), mxGetPr(prhs[1]) + (numel(prhs[1]) - (mwSize)N), mxGetPr(plhs[0]));
  if (rc) { mxDestroyArray(plhs[0]); plhs[0] = NULL; sb_check(rc, "psdinvscale"); }
}
