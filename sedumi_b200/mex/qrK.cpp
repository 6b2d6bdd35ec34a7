// [q,r] = qrK(x,K)   Householder QR of every PSD block, q in SeDuMi's product form   (qrK.c:239-297)
#include "mex_common.h"

void mexFunction(int nlhs, mxArray *plhs[], int nrhs, const mxArray *prhs[]) {
  MEX_REQUIRE(nrhs >= 2, "qrK requires more input arguments");
  MEX_REQUIRE(nlhs <= 2, "qrK produces less output arguments");
  ConeK K;
  read_cone(prhs[1], K);
  MEX_REQUIRE(K.rsdpN == K.sdpN, "qrK: Hermitian PSD blocks are not handled by the CUDA plugin");
  const sb_idx sdpdim = K.rDim + K.hDim;
  MEX_REQUIRE((sb_idx)numel(prhs[0]) == sdpdim, "size mismatch x");
  mxArray *Q = mxCreateDoubleMatrix((mwSize)(sdpdim + K.hLen), 1, mxREAL), *R = mxCreateDoubleMatrix((mwSize)sdpdim, 1, mxREAL);
  int rc = sb200_qrK(K.sdpN, K.s.data(), mxGetPr(prhs[0]), mxGetPr(Q), mxGetPr(R));
  if (rc) { mxDestroyArray(Q); mxDestroyArray(R); sb_check(rc, "qrK"); }
  plhs[0] = Q;
  if (nlhs >= 2) plhs[1] = R; else mxDestroyArray(R);
}
