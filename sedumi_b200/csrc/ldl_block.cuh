// ldl_block.cuh -- the 32 x 32 diagonal block of an LDL' panel, factored by one warp in registers with SeDuMi's pivot
// rules (blkchol2.c:96-167); shared by the dense single-supernode kernel (chol_dense.cu) and the supernodal one (chol.cu).
#pragma once

namespace sb {

static const int LDLB = 32;

// The 32 x 32 diagonal block, factored by ONE warp with the block in registers: lane r holds row r as a window a[j] =
// A[r][k+j] that slides one column per pivot, so every register index is static while the pivot loop itself stays a
// loop (fully unrolled, the 496 shuffle/FMA pairs were 20 000 instructions -- more than the instruction cache -- and
// ran slower than the shared-memory version).  The pivot column travels by shuffles; a step has no barrier.
// A separate, non-inlined function so that the window gets registers of its own.  Returns the first pivot that needs
// the reference's stability test (w if none); the state up to there is written back to A / dloc / skipped.
static __device__ __noinline__ int warp_factor_block(double (*A)[LDLB + 1], const double *s_lb, double *dloc, int *skipped, int *flag,
                                              double *sval, int p0, int w, int m, double ub, int k_resume, int resolved_k, double s_x) {
  const int lane = threadIdx.x & 31;
  double a[LDLB];
#pragma unroll
  for (int j = 0; j < LDLB; j++) a[j] = (k_resume + j < LDLB) ? A[lane][k_resume + j] : 0.0;
  int k = k_resume;
  for (; k < w; k++) {
    const int gk = p0 + k;
    double xkk = __shfl_sync(0xffffffffu, a[0], k);
    const bool resolved = (k == resolved_k);
    if (resolved) xkk = s_x;
    const bool skip = !(xkk > s_lb[k]);
    if (!skip && !resolved && (m - gk > 1) && (xkk < ub)) break;        // stability test needed (uniform)
    if (skip) {
      if (lane == 0) { flag[gk] = 1; sval[gk] = xkk; skipped[k] = 1; dloc[k] = 0.0; }
      if (lane >= k) A[lane][k] = a[0];                                 // the column is left as it is
    } else {
      const double rinv = 1.0 / xkk;
      const double xr = (lane > k) ? a[0] : 0.0;
      // element (r, c = k+j), k < c <= r: A[r][c] -= (A[c][k]/xkk) * A[r][k]
#pragma unroll
      for (int j = 1; j < LDLB; j++) {
        const double ack = __shfl_sync(0xffffffffu, a[0], min(k + j, LDLB - 1));
        if (k + j < LDLB && lane >= k + j) a[j] -= (ack * rinv) * xr;
      }
      if (lane > k) A[lane][k] = a[0] * rinv;
      if (lane == k) { A[k][k] = 1.0; dloc[k] = xkk; }
    }
#pragma unroll
    for (int j = 0; j + 1 < LDLB; j++) a[j] = a[j + 1];
    a[LDLB - 1] = 0.0;
  }
  if (k < w) {                                                           // stopped: hand the updated columns back
#pragma unroll
    for (int j = 0; j < LDLB; j++) if (k + j < LDLB) A[lane][k + j] = a[j];
  }
  return k;
}


// The same for an 8 x 8 diagonal block, fully unrolled and branch-free (lanes 0..7 hold the rows): 28 shuffle / FMA
// steps.  Used by the supernodal panel kernel, whose blocked pass advances 8 columns at a time -- the 32-wide version
// above costs ~1 600 instructions per pivot on a single warp (sliding-window moves, predicated selects and a
// WARPSYNC/ENDCOLLECTIVE pair around every shuffle).
static const int LDLS = 8;
static __device__ __forceinline__ int warp_factor_block8(double (*A)[LDLS + 1], const double *s_lb, double *dloc, int *skipped, int *flag,
                                                         double *sval, int p0, int w, int m, double ub) {
  const int lane = threadIdx.x & 31;
  double a[LDLS];
#pragma unroll
  for (int c = 0; c < LDLS; c++) a[c] = (lane < LDLS) ? A[lane][c] : 0.0;
  int kstop = w;
#pragma unroll
  for (int k = 0; k < LDLS; k++) {
    const double xkk = __shfl_sync(0xffffffffu, a[k], k);
    const bool live = (k < w) && (kstop == w);
    const bool skip = !(xkk > s_lb[k]);
    const bool trig = live && !skip && (m - (p0 + k) > 1) && (xkk < ub);
    if (trig) kstop = k;                                     // uniform: every lane sees the same xkk
    const bool upd = live && !skip && !trig;
    if (live && skip && lane == 0) { flag[p0 + k] = 1; sval[p0 + k] = xkk; skipped[k] = 1; dloc[k] = 0.0; }
    const double rinv = upd ? 1.0 / xkk : 0.0;
    const double xr = (lane > k) ? a[k] : 0.0;
#pragma unroll
    for (int c = k + 1; c < LDLS; c++) {
      const double ack = __shfl_sync(0xffffffffu, a[k], c);
      if (upd && lane >= c) a[c] -= (ack * rinv) * xr;
    }
    if (upd && lane > k) a[k] *= rinv;
    if (upd && lane == k) { a[k] = 1.0; dloc[k] = xkk; }
  }
  if (lane < LDLS) {
#pragma unroll
    for (int c = 0; c < LDLS; c++) A[lane][c] = a[c];
  }
  return kstop;
}

}  // namespace sb
