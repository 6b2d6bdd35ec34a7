// z = triumtriu(x,y,K)   (triumtriu.m: M code in the reference; a MEX of the same name shadows it)
#include "mex_common.h"

void mexFunction(int nlhs, mxArray *plhs[], int nrhs, const mxArray *prhs[]) {
  MEX_REQUIRE(nrhs >= 3, "triumtriu requires 3 input arguments.");
  MEX_REQUIRE(nlhs <= 1, "triumtriu generates 1 output argument.");
  ConeK K;
  read_cone(prhs[2], K);
  if (K.sdpN == 0) { plhs[0] = mxCreateDoubleMatrix(0, 0, mxREAL); return; }
  MEX_REQUIRE(K.rsdpN == K.sdpN, "triumtriu: Hermitian PSD blocks are not handled by the CUDA plugin");
  const sb_idx N = K.rDim;
  MEX_REQUIRE((sb_idx)numel(prhs[0]) >= N && numel(prhs[1]) == numel(prhs[0]), "x/y size mismatch");
  MEX_REQUIRE(!mxIsSparse(prhs[0]) && !mxIsSparse(prhs[1]), "x and y must be full");
  const mwSize skip = numel(prhs[0]) - (mwSize)N;                      // the PSD part is the tail (xi = length(x) - N)
  plhs[0] = mxCreateDoubleMatrix((mwSize)N, 1, mxREAL);
  int rc = sb200_psdmul(1, K.sdpN, K.s.data(), mxGetPr(prhs[0]) + skip, mxGetPr(prhs[1]) + skip, mxGetPr(plhs[0]));
  if (rc) { mxDestroyArray(plhs[0]); plhs[0] = NULL; sb_check(rc, "triumtriu"); }
}
