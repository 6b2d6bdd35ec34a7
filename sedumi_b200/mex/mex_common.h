// mex_common.h -- helpers shared by the CUDA MEX stubs.  The stubs contain no arithmetic:
// they validate like the reference's debug build (mxAssert -> mexErrMsgTxt), unpack
// mxArrays into the plain pointers of include/sedumi_b200.h and build the outputs with the
// reference's exact layout.  They compile unchanged against MATLAB's / Octave's mex.h.
#pragma once
#include <math.h>
#include <stdio.h>
#include <string.h>
#include <vector>
#include "mex.h"
#include "sedumi_b200.h"

#define MEX_REQUIRE(cond, msg) do { if (!(cond)) mexErrMsgTxt(msg); } while (0)

// Library failures surface as MATLAB errors, never exit() (SURVEY.md section 8b).
static inline void sb_check(int rc, const char *who) {
  if (rc != 0) {
    static char buf[1200];
    snprintf(buf, sizeof buf, "%s: %s", who, sb200_last_error());
    mexErrMsgTxt(buf);
  }
}

static inline mwSize numel(const mxArray *a) { return mxGetM(a) * mxGetN(a); }

// 1-based (or 0-based if base==0) double index vector -> 0-based int64
static inline void idx_from_double(const mxArray *a, std::vector<sb_idx> &out, int base, const char *what) {
  mwSize n = numel(a);
  const double *p = mxGetPr(a);
  out.resize(n);
  for (mwSize i = 0; i < n; i++) {
    double v = p[i] - base;
    if (!(v >= 0) || v != floor(v)) {
      static char buf[256];
      snprintf(buf, sizeof buf, "%s must hold %s integers.", what, base ? "positive" : "nonnegative");
      mexErrMsgTxt(buf);
    }
    out[i] = (sb_idx)v;
  }
}

// mwIndex (size_t) arrays are bit-compatible with sb_idx (int64) on 64-bit platforms.
static inline const sb_idx *as_idx(const mwIndex *p) {
  static_assert(sizeof(mwIndex) == sizeof(sb_idx), "mwIndex must be 64-bit");
  return reinterpret_cast<const sb_idx *>(p);
}

static inline const mxArray *need_field(const mxArray *s, const char *name, const char *msg) {
  const mxArray *f = mxGetField(s, 0, name);
  if (!f) mexErrMsgTxt(msg);
  return f;
}

// Cone description as conepars() reads it (sdmauxCone.c:48-134).
struct ConeK {
  sb_idx lpN = 0, lorN = 0, sdpN = 0, rsdpN = 0;
  std::vector<sb_idx> q, s;         // Lorentz orders, PSD orders
  sb_idx qDim = 0, rDim = 0, hDim = 0, rLen = 0, hLen = 0;
};
static inline void read_cone(const mxArray *mxK, ConeK &K) {
  MEX_REQUIRE(mxIsStruct(mxK), "Parameter `K' should be a structure.");
  const mxArray *f;
  if ((f = mxGetField(mxK, 0, "l")) != NULL) K.lpN = (sb_idx)mxGetScalar(f);
  if ((f = mxGetField(mxK, 0, "q")) != NULL) {
    mwSize n = numel(f); const double *p = mxGetPr(f);
    if (!(n == 1 && p[0] == 0.0)) for (mwSize i = 0; i < n; i++) K.q.push_back((sb_idx)p[i]);
  }
  if ((f = mxGetField(mxK, 0, "s")) != NULL) {
    mwSize n = numel(f); const double *p = mxGetPr(f);
    if (!(n == 1 && p[0] == 0.0)) for (mwSize i = 0; i < n; i++) K.s.push_back((sb_idx)p[i]);
  }
  K.lorN = (sb_idx)K.q.size();
  K.sdpN = (sb_idx)K.s.size();
  K.rsdpN = K.sdpN;
  if ((f = mxGetField(mxK, 0, "rsdpN")) != NULL) K.rsdpN = (sb_idx)mxGetScalar(f);
  MEX_REQUIRE(K.rsdpN <= K.sdpN, "K.rsdpN mismatches K.s");
  for (sb_idx i = 0; i < K.lorN; i++) K.qDim += K.q[i];
  for (sb_idx i = 0; i < K.sdpN; i++) {
    if (i < K.rsdpN) { K.rDim += K.s[i] * K.s[i]; K.rLen += K.s[i]; }
    else { K.hDim += 2 * K.s[i] * K.s[i]; K.hLen += K.s[i]; }
  }
}

// A sparse m x n output with the pattern (jc, ir) and UNINITIALISED values: the index and value arrays come from
// mxMalloc and are attached with mxSetIr/mxSetPr/mxSetNzmax (documented MEX API), so that a multi-megabyte output
// (ADA, L.L) is not zero-filled by mxCreateSparse before it is overwritten.
static inline mxArray *sparse_with_pattern(mwSize m, mwSize n, const mwIndex *jc, const mwIndex *ir) {
  const mwSize nnz = jc[n], cap = nnz ? nnz : 1;
  mxArray *a = mxCreateSparse(m, n, 1, mxREAL);
  mxFree(mxGetPr(a));
  mxFree(mxGetIr(a));
  mwIndex *nir = (mwIndex *)mxMalloc(cap * sizeof(mwIndex));
  double *npr = (double *)mxMalloc(cap * sizeof(double));
  if (!nir || !npr) mexErrMsgTxt("Memory allocation error.");
  mxSetIr(a, nir);
  mxSetPr(a, npr);
  mxSetNzmax(a, cap);
  memcpy(mxGetJc(a), jc, (n + 1) * sizeof(mwIndex));
  memcpy(nir, ir, nnz * sizeof(mwIndex));
  if (!nnz) { nir[0] = 0; npr[0] = 0.0; }
  return a;
}
