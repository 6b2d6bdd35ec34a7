// mineig = minpsdeig(x,K)   smallest spectral coefficient over all PSD blocks (minpsdeig.m:43-68; M code in the reference)
#include <vector>
#include "mex_common.h"

void mexFunction(int nlhs, mxArray *plhs[], int nrhs, const mxArray *prhs[]) {
  MEX_REQUIRE(nrhs >= 2, "minpsdeig requires 2 input arguments.");
  MEX_REQUIRE(nlhs <= 1, "minpsdeig generates 1 output argument.");
  ConeK K;
  read_cone(prhs[1], K);
  if (K.sdpN == 0) { plhs[0] = mxCreateDoubleMatrix(0, 0, mxREAL); return; }
  MEX_REQUIRE(K.rsdpN == K.sdpN, "minpsdeig: Hermitian PSD blocks are not handled by the CUDA plugin");
  const sb_idx N = K.rDim;
  MEX_REQUIRE((sb_idx)numel(prhs[0]) >= N, "x size mismatch");
  MEX_REQUIRE(!mxIsSparse(prhs[0]), "x must be full");
  std::vector<double> lab((size_t)K.rLen);
  sb_check(sb200_psdeig(K.sdpN, K.s.data(), mxGetPr(prhs[0]) + (numel(prhs[0]) - (mwSize)N), lab.data(), NULL), "minpsdeig");
  double mn = lab[0];
  for (double v : lab) mn = v < mn ? v : mn;
  plhs[0] = mxCreateDoubleMatrix(1, 1, mxREAL);
  mxGetPr(plhs[0])[0] = mn;
}
