// chol.cu -- supernodal sparse LDL' on H100: numeric factorisation with SeDuMi's pivot
// safeguards, and the forward/backward block solves.
//
// Reference semantics reproduced (not its code structure):
//   blkchol.c:95-120   permuteP   L := tril(X(perm,perm)) on the symbolic pattern
//   blkchol.c:157-231  spchol     ub = max diag / maxu^2, lb = max(abstol, canceltol*absd(perm))
//   blkchol2.c:96-167  cholonBlk  skip pivot if x_kk <= lb_k (d_k = 0, column left alone);
//                                 if x_kk < ub, compare with a sub-column magnitude / maxu
//                                 and raise the pivot to it ("diag add")
//   blkchol2.c:346-420 precorrect updates from earlier supernodes, skipped columns excluded
//   fwblkslv.c:77-134 / bwblkslv.c:73-125  dense-RHS block solves
//
// GPU design.  The reference is a sequential left-looking supernodal code driven by linked
// lists.  Here the symbolic structure is compiled once into a *plan*: supernode panels in a
// rectangular column-major layout, the list of (descendant K -> ancestor J) update pairs
// with precomputed relative row positions, and a level schedule of the supernodal
// elimination tree.  Numeric work per level = one batched "pull" update kernel (each CTA owns
// a tile of an ancestor panel and subtracts the contributions of all its descendants in a
// fixed order -> deterministic, no atomics) + factor kernels.  Supernodes up to SMALL_N
// columns are factored by one CTA each (batched across the level); wider ones use a blocked
// right-looking scheme (diag-block CTA with the pivot rules, row-parallel triangular solve,
// tiled FP64 trailing update).
//
// A note on the "diag add" threshold: the reference evaluates
//     ubk = fabs(x[idamax(...)]) / maxu                       (blkchol2.c:66-70,122)
// with a Fortran (1-based) idamax used as a C index, so the magnitude actually read is the
// element FOLLOWING the first maximum of the sub-column (for a maximum in the last row: the
// first element of the next packed column, i.e. the next pivot's current diagonal).  That
// is what every build of the reference against a conforming BLAS computes, so it is what
// we reproduce (see next_after_first_max below); DESIGN.md discusses it.
#include <algorithm>
#include <map>
#include <math.h>
#include <stdlib.h>
#include <time.h>
#include "sb_internal.h"

#include "chol_plan.h"
#include "ldl_block.cuh"

namespace sb {

// ======================================================================= device helpers
struct ArgMax { double v; int i; };
__device__ __forceinline__ ArgMax am_better(ArgMax a, ArgMax b) {
  // first element of maximum magnitude (idamax semantics: ties -> smallest index)
  if (b.v > a.v || (b.v == a.v && b.i < a.i)) return b;
  return a;
}
__device__ __forceinline__ ArgMax block_argmax(ArgMax x, ArgMax *sh) {
  for (int o = 16; o > 0; o >>= 1) {
    ArgMax y; y.v = __shfl_down_sync(0xffffffffu, x.v, o); y.i = __shfl_down_sync(0xffffffffu, x.i, o);
    x = am_better(x, y);
  }
  int w = threadIdx.x >> 5, l = threadIdx.x & 31, nw = (blockDim.x + 31) >> 5;
  __syncthreads();
  if (l == 0) sh[w] = x;
  __syncthreads();
  if (w == 0) {
    x = (l < nw) ? sh[l] : ArgMax{-1.0, 0x7fffffff};
    for (int o = 16; o > 0; o >>= 1) {
      ArgMax y; y.v = __shfl_down_sync(0xffffffffu, x.v, o); y.i = __shfl_down_sync(0xffffffffu, x.i, o);
      x = am_better(x, y);
    }
    if (l == 0) sh[0] = x;
  }
  __syncthreads();
  x = sh[0];
  __syncthreads();
  return x;
}

// ======================================================================= permuteP
// One CTA per column j of L: gathers X(perm(rows), perm(j)) into the rect panel.
__global__ void permuteP_kernel(const Sn *sn, const int *snode, const int *lindx, const int *perm,
                                const int *Xjc, const int *Xir, const double *Xpr,
                                double *rect, double *diagX) {
  int j = blockIdx.x;
  Sn s = sn[snode[j]];
  int c = j - s.first;
  const int *rows = lindx + s.lindx;
  double *col = rect + s.poff + (long long)c * s.m;
  int pj = perm[j];
  int b0 = Xjc[pj], b1 = Xjc[pj + 1];
  bool dense = (b1 - b0) == (int)gridDim.x;       // full column: row r sits at b0 + r
  for (int t = threadIdx.x; t < s.m; t += blockDim.x) {
    double v = 0.0;
    if (t >= c) {
      int pi = perm[rows[t]];
      if (dense) v = Xpr[b0 + pi];
      else {
        int lo = b0, hi = b1;
        while (lo < hi) { int mid = (lo + hi) >> 1; if (Xir[mid] < pi) lo = mid + 1; else hi = mid; }
        if (lo < b1 && Xir[lo] == pi) v = Xpr[lo];
      }
      if (t == c) diagX[j] = v;
    }
    col[t] = v;
  }
}

// scal[0] = ub = max(diag)/maxu^2 ; lb[j] = max(abstol, canceltol * (absd ? absd[perm[j]] : diag[j]))
__global__ void bounds_kernel(int m, const double *diagX, const double *absd, const int *perm,
                              double abstol, double canceltol, double maxu, double *lb, double *scal) {
  __shared__ double sh[32];
  double mx = 0.0;
  for (int j = threadIdx.x; j < m; j += blockDim.x) {
    double dj = diagX[j];
    if (dj > mx) mx = dj;
    double o = canceltol * (absd ? absd[perm[j]] : dj);
    lb[j] = (o > abstol) ? o : abstol;
  }
  for (int o = 16; o > 0; o >>= 1) mx = fmax(mx, __shfl_down_sync(0xffffffffu, mx, o));
  if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = mx;
  __syncthreads();
  if (threadIdx.x < 32) {
    mx = (threadIdx.x < ((blockDim.x + 31) >> 5)) ? sh[threadIdx.x] : 0.0;
    for (int o = 16; o > 0; o >>= 1) mx = fmax(mx, __shfl_down_sync(0xffffffffu, mx, o));
    if (threadIdx.x == 0) scal[0] = mx / (maxu * maxu);
  }
}

// ======================================================================= update (pull)
// CTA = one UT_R x UT_C tile of ancestor panel J; loops over J's descendants in order.
__global__ void __launch_bounds__(256)
update_kernel(const UTile *tiles, const Sn *sn, const Pair *pairs, const int *pair_beg,
              const int *rel, const double *U, double *rect) {
  UTile tl = tiles[blockIdx.x];
  Sn sj = sn[tl.J];
  double *PJ = rect + sj.poff;
  int r0 = tl.r0, r1 = min(tl.r0 + UT_R, sj.m), c0 = tl.c0, c1 = min(tl.c0 + UT_C, sj.n);
  // The sub-range of every descendant that falls into this tile is found first, one descendant per thread (the
  // bisections are chains of dependent global loads: done one descendant at a time by a single thread they cost more
  // than the update itself); then the descendants are applied in list order, one block barrier each (two descendants
  // may hit the same entry from different threads).
  __shared__ int4 s_rng[256];
  const int pb = pair_beg[tl.J], pe = pair_beg[tl.J + 1];
  for (int e0 = pb; e0 < pe; e0 += 256) {
    const int ne = min(256, pe - e0);
    __syncthreads();
    if (threadIdx.x < ne) {
      const Pair p = pairs[e0 + threadIdx.x];
      const int *rl = rel + p.rel;
      int4 g;
      int lo = 0, hi = p.mk;
      while (lo < hi) { int mid = (lo + hi) >> 1; if (rl[mid] < r0) lo = mid + 1; else hi = mid; }
      g.x = lo; hi = p.mk;
      while (lo < hi) { int mid = (lo + hi) >> 1; if (rl[mid] < r1) lo = mid + 1; else hi = mid; }
      g.y = lo;
      lo = 0; hi = p.ncolup;
      while (lo < hi) { int mid = (lo + hi) >> 1; if (rl[mid] < c0) lo = mid + 1; else hi = mid; }
      g.z = lo; hi = p.ncolup;
      while (lo < hi) { int mid = (lo + hi) >> 1; if (rl[mid] < c1) lo = mid + 1; else hi = mid; }
      g.w = lo;
      s_rng[threadIdx.x] = g;
    }
    __syncthreads();
    for (int i = 0; i < ne; i++) {
      const int4 g = s_rng[i];
      const int nr = g.y - g.x, nc = g.w - g.z;
      if (nr <= 0 || nc <= 0) continue;                // uniform
      const Pair p = pairs[e0 + i];
      const int *rl = rel + p.rel;
      const Sn sk = sn[p.K];
      const int mk = sk.m - sk.n, u0 = p.koff - sk.n;  // U_K is indexed by K's rows below its diagonal block
      const double *UK = U + sk.uoff;
      for (int idx = threadIdx.x; idx < nr * nc; idx += blockDim.x) {
        const int t1 = g.x + idx % nr, t2 = g.z + idx / nr;
        if (t1 < t2) continue;                         // strictly above the diagonal of J
        PJ[rl[t1] + (long long)rl[t2] * sj.m] -= UK[(u0 + t1) + (long long)(u0 + t2) * mk];
      }
      __syncthreads();
    }
  }
}

// The same update through the plan's gather lists: a thread owns an entry of the ancestor panel and sums the entries of
// the contribution blocks that reach it, in descendant order (deterministic; no barrier, no search).
__global__ void __launch_bounds__(256)
update_gather_kernel(const UTile *tiles, const Sn *sn, const int *uptr, const long long *usrc, const int *uK,
                     const unsigned char *kmask, const double *U, double *rect) {
  const UTile tl = tiles[blockIdx.x];
  const Sn sj = sn[tl.J];
  const int r0 = tl.r0, r1 = min(tl.r0 + UT_R, sj.m), c0 = tl.c0, c1 = min(tl.c0 + UT_C, sj.n);
  const int nr = r1 - r0, nc = c1 - c0;
  for (int idx = threadIdx.x; idx < nr * nc; idx += blockDim.x) {
    const int r = r0 + idx % nr, c = c0 + idx / nr;
    if (r < c) continue;
    const long long e = sj.poff + r + (long long)c * sj.m;
    double acc = 0.0;
    for (int q = uptr[e]; q < uptr[e + 1]; q++) if (!kmask || kmask[uK[q]]) acc += U[usrc[q]];
    rect[e] -= acc;
  }
}

// ======================================================================= Schur contributions
// U_K = L21 D L21' (lower triangle) for every supernode of a list: blockIdx.x = supernode, blockIdx.y = lower 64x64
// tile.  Skipped pivots have d = 0 and drop out (blkchol2.c:375,389).
__global__ void __launch_bounds__(256)
schur_kernel(const int *list, const Sn *sn, const double *rect, const double *d, double *U) {
  const Sn s = sn[list[blockIdx.x]];
  const int mk = s.m - s.n;
  if (mk <= 0) return;
  const int nt = (mk + 63) / 64;
  int t = blockIdx.y;
  if (t >= nt * (nt + 1) / 2) return;
  int ti = 0;
  while (t > ti) { t -= ti + 1; ti++; }
  const int r0 = ti * 64, c0 = t * 64;
  __shared__ double As[16][64 + 1], Bs[16][64 + 1];
  const double *P = rect + s.poff + s.n;
  const double *dk = d + s.first;
  const int ld = s.m;
  const int tx = threadIdx.x % 16, ty = threadIdx.x / 16;
  double acc[4][4] = {};
  for (int k0 = 0; k0 < s.n; k0 += 16) {
    for (int idx = threadIdx.x; idx < 64 * 16; idx += blockDim.x) {
      const int i = idx % 64, j = idx / 64, kk = k0 + j;
      const bool in = kk < s.n;
      As[j][i] = (in && r0 + i < mk) ? P[(long long)kk * ld + r0 + i] : 0.0;
      Bs[j][i] = (in && c0 + i < mk) ? P[(long long)kk * ld + c0 + i] * dk[kk] : 0.0;
    }
    __syncthreads();
#pragma unroll
    for (int j = 0; j < 16; j++) {
      double av[4], bv[4];
#pragma unroll
      for (int i = 0; i < 4; i++) { av[i] = As[j][tx + 16 * i]; bv[i] = Bs[j][ty + 16 * i]; }
#pragma unroll
      for (int i = 0; i < 4; i++)
#pragma unroll
        for (int q = 0; q < 4; q++) acc[i][q] += av[i] * bv[q];
    }
    __syncthreads();
  }
  double *UK = U + s.uoff;
#pragma unroll
  for (int q = 0; q < 4; q++) {
    const int c = c0 + ty + 16 * q;
    if (c >= mk) continue;
#pragma unroll
    for (int i = 0; i < 4; i++) {
      const int r = r0 + tx + 16 * i;
      if (r < mk && r >= c) UK[r + (long long)c * mk] = acc[i][q];
    }
  }
}

// ======================================================================= small supernodes
// One CTA factors one whole supernode panel (m x n), column by column; the panel is staged in shared memory when it
// fits (cap doubles), otherwise worked on in place (L2).
__global__ void __launch_bounds__(512)
factor_small_kernel(const int *list, const Sn *sn, double *rect, double *d, const double *lb,
                    const double *scal, double maxu, int *flag, double *sval,
                    const double *diagX, int mtot, int cap) {
  extern __shared__ __align__(16) double pan[];
  __shared__ __align__(8) unsigned long long pan_bar;
  Sn s = sn[list[blockIdx.x]];
  double *Pg = rect + s.poff;
  const int ld = s.m, n = s.n, m = s.m;
  const bool insm = (long long)m * n <= cap;
  double *P = Pg;
  // The panel is one contiguous, 16-byte aligned run of m*n doubles (padded to an even count): it is staged into shared
  // memory by the TMA unit as 1-D bulk copies that complete on an mbarrier, and written back the same way.
  const unsigned pan_bytes = (unsigned)((((long long)m * n + 1) & ~1LL) * 8);
  if (insm) {
    const unsigned bar = (unsigned)__cvta_generic_to_shared(&pan_bar), dst = (unsigned)__cvta_generic_to_shared(pan);
    if (threadIdx.x == 0) {
      asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;\n" :: "r"(bar) : "memory");
      asm volatile("fence.mbarrier_init.release.cluster;\n" ::: "memory");
      asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;\n" :: "r"(bar), "r"(pan_bytes) : "memory");
      for (unsigned off = 0; off < pan_bytes; off += 65536u) {
        const unsigned len = min(65536u, pan_bytes - off);
        asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];\n"
                     :: "r"(dst + off), "l"((const char *)Pg + off), "r"(len), "r"(bar) : "memory");
      }
    }
    __syncthreads();                                   // the barrier is initialised before anybody waits on it
    asm volatile("{\n .reg .pred P1;\n LAB_WAIT:\n mbarrier.try_wait.parity.shared::cta.b64 P1, [%0], 0;\n @P1 bra DONE;\n bra LAB_WAIT;\n DONE:\n }\n"
                 :: "r"(bar) : "memory");
    P = pan;
  }
  const double ub = scal[0];
  __shared__ ArgMax sh_am[32];
  __shared__ double s_x;
  // ---- blocked pass: 8 columns at a time.  The diagonal block is factored by one warp in registers (ldl_block.cuh),
  // every row below it is brought up to date by its own thread (an 8-step substitution in registers) and the rest of
  // the panel takes the rank-8 update, one warp per column.  A pivot that needs the reference's stability test (rare)
  // ends the blocked pass: the remaining columns, starting with this block, go through the column-by-column code
  // below, which evaluates the test on the fully updated column exactly like cholonBlk.
  __shared__ double Ab[LDLS][LDLS + 1];
  __shared__ double b_lb[LDLS], b_d[LDLS], b_rd[LDLS];
  __shared__ int b_skip[LDLS], b_stop;
  int kleg = 0;                                        // first column left to the column-by-column code
  for (int p0 = 0; p0 < n; p0 += LDLS) {
    const int w = min(LDLS, n - p0);
    if (threadIdx.x < LDLS * LDLS) {
      const int r = threadIdx.x % LDLS, c = threadIdx.x / LDLS;
      Ab[r][c] = (r < w && c < w && r >= c) ? P[(long long)(p0 + c) * ld + p0 + r] : 0.0;
    }
    if (threadIdx.x < LDLS) { b_skip[threadIdx.x] = 0; b_d[threadIdx.x] = 0.0; b_lb[threadIdx.x] = threadIdx.x < w ? lb[s.first + p0 + threadIdx.x] : 0.0; }
    __syncthreads();
    if (threadIdx.x < 32) {
      // global column = s.first + p0 + k; "column longer than 1" <=> (s.first + m) - (s.first + p0 + k) > 1
      const int ks = warp_factor_block8(Ab, b_lb, b_d, b_skip, flag, sval, s.first + p0, w, s.first + m, ub);
      if (threadIdx.x == 0) b_stop = ks;
    }
    __syncthreads();
    if (b_stop < w) {                                  // undo the marks of this block and leave the rest to the column code
      if (threadIdx.x < w && b_skip[threadIdx.x]) { flag[s.first + p0 + threadIdx.x] = 0; sval[s.first + p0 + threadIdx.x] = 0.0; }
      kleg = p0;
      break;
    }
    kleg = p0 + w;
    if (threadIdx.x < LDLS) b_rd[threadIdx.x] = (threadIdx.x < w && b_d[threadIdx.x] > 0.0) ? 1.0 / b_d[threadIdx.x] : 0.0;
    if (threadIdx.x < w) d[s.first + p0 + threadIdx.x] = b_d[threadIdx.x];
    // L11 back into the panel (unit lower; a skipped column keeps no entries below its diagonal)
    if (threadIdx.x < w * w) {
      const int r = threadIdx.x % w, c = threadIdx.x / w;
      if (r >= c) P[(long long)(p0 + c) * ld + p0 + r] = (r == c) ? 1.0 : (b_skip[c] ? 0.0 : Ab[r][c]);
    }
    __syncthreads();
    // rows below the block: L21 = A21 L11^-T D^-1, one thread per row
    for (int r = p0 + w + threadIdx.x; r < m; r += blockDim.x) {
      double a[LDLS];
#pragma unroll
      for (int j = 0; j < LDLS; j++) a[j] = (j < w) ? P[(long long)(p0 + j) * ld + r] : 0.0;
#pragma unroll
      for (int j = 0; j < LDLS; j++) {
        const double rj = b_rd[j];
        const double xj = a[j];
        if (rj > 0.0) {
#pragma unroll
          for (int j2 = j + 1; j2 < LDLS; j2++) a[j2] -= xj * Ab[j2][j];
          a[j] = xj * rj;
        } else a[j] = 0.0;
      }
#pragma unroll
      for (int j = 0; j < LDLS; j++) if (j < w) P[(long long)(p0 + j) * ld + r] = a[j];
    }
    __syncthreads();
    // rank-w update of the remaining columns of the panel: P(r,c) -= sum_j L(r,j) d_j L(c,j), r >= c > last block column.
    // One warp per column, lanes over rows; the column's scaled entries are broadcast reads.
    {
      const int c0 = p0 + w, warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = blockDim.x >> 5;
      for (int c = c0 + warp; c < n; c += nw) {
        double *cc = P + (long long)c * ld;
        double lc[LDLS];
#pragma unroll
        for (int j = 0; j < LDLS; j++) lc[j] = (j < w) ? b_d[j] * P[(long long)(p0 + j) * ld + c] : 0.0;
        for (int r = c + lane; r < m; r += 32) {
          double acc = 0.0;
#pragma unroll
          for (int j = 0; j < LDLS; j++) if (j < w) acc += P[(long long)(p0 + j) * ld + r] * lc[j];
          cc[r] -= acc;
        }
      }
    }
    __syncthreads();
  }
  for (int k = kleg; k < n; k++) {
    const int gk = s.first + k;
    double *ck = P + (long long)k * ld;
    double xkk = ck[k];
    double lbk = lb[gk];
    bool skip = !(xkk > lbk);
    bool trig = !skip && (m - k > 1) && (xkk < ub);      // uniform across the CTA
    if (trig) {
      ArgMax am{-1.0, 0x7fffffff};
      for (int t = k + 1 + threadIdx.x; t < m; t += blockDim.x) am = am_better(am, ArgMax{fabs(ck[t]), t});
      am = block_argmax(am, sh_am);
      if (threadIdx.x == 0) {
        int t = am.i + 1;                                // element following the first maximum
        double v;
        if (t < m) v = ck[t];
        else if (k + 1 < n) v = P[(long long)(k + 1) * ld + (k + 1)];
        else v = (gk + 1 < mtot) ? diagX[gk + 1] : 0.0;
        double ubk = fabs(v) / maxu;
        if (xkk < ubk) { flag[gk] = 2; sval[gk] = ubk - xkk; xkk = ubk; }
        s_x = xkk;
      }
      __syncthreads();
      xkk = s_x;
      __syncthreads();
    }
    if (skip) {
      if (threadIdx.x == 0) { d[gk] = 0.0; flag[gk] = 1; sval[gk] = xkk; }
      continue;                                          // column untouched, excluded from updates
    }
    // right-looking update of the remaining columns of the supernode with the UNDIVIDED column
    const int ncol = n - k - 1;
    if (ncol > 0) {
      // warp per column c, lanes over rows
      int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = blockDim.x >> 5;
      for (int c = k + 1 + warp; c < n; c += nw) {
        double lck = ck[c] / xkk;
        double *cc = P + (long long)c * ld;
        for (int r = c + lane; r < m; r += 32) cc[r] -= lck * ck[r];
      }
    }
    __syncthreads();
    for (int r = k + 1 + threadIdx.x; r < m; r += blockDim.x) ck[r] /= xkk;
    if (threadIdx.x == 0) { d[gk] = xkk; ck[k] = 1.0; }
    __syncthreads();
  }
  if (insm) {
    __syncthreads();
    if (threadIdx.x == 0) {
      asm volatile("fence.proxy.async.shared::cta;\n" ::: "memory");     // generic-proxy writes of the panel -> visible to the bulk store
      const unsigned src = (unsigned)__cvta_generic_to_shared(pan);
      for (unsigned off = 0; off < pan_bytes; off += 65536u) {
        const unsigned len = min(65536u, pan_bytes - off);
        asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;\n" :: "l"((char *)Pg + off), "r"(src + off), "r"(len) : "memory");
      }
      asm volatile("cp.async.bulk.commit_group;\n" ::: "memory");
      asm volatile("cp.async.bulk.wait_group 0;\n" ::: "memory");
    }
  }
}

// ======================================================================= blocked path
// diag kernel: factor the w x w diagonal block at panel offset p0 of supernode S.
// Tail rows (below the block) are only needed when the stability test fires.
__global__ void __launch_bounds__(256)
diag_kernel(Sn s, int p0, int w, double *rect, double *d, const double *lb, const double *scal,
            double maxu, int *flag, double *sval, const double *diagX, int mtot, double *vscratch) {
  __shared__ double A[NB][NB + 1];
  __shared__ double z[NB], dloc[NB];
  __shared__ int skipped[NB];
  __shared__ ArgMax sh_am[32];
  __shared__ double s_x;
  double *P = rect + s.poff;
  const int ld = s.m, m = s.m, n = s.n;
  const double ub = scal[0];
  for (int idx = threadIdx.x; idx < w * w; idx += blockDim.x) {
    int r = idx % w, c = idx / w;
    A[r][c] = (r >= c) ? P[(long long)(p0 + c) * ld + p0 + r] : 0.0;
  }
  if (threadIdx.x < NB) { skipped[threadIdx.x] = 0; dloc[threadIdx.x] = 0.0; }
  __syncthreads();
  for (int k = 0; k < w; k++) {
    const int gk = s.first + p0 + k;
    double xkk = A[k][k];
    double lbk = lb[gk];
    bool skip = !(xkk > lbk);
    const int collen = m - (p0 + k);                     // remaining length incl. diagonal
    bool trig = !skip && (collen > 1) && (xkk < ub);
    if (trig) {
      // z: last column of (I+S)^-1, so that  v_tail = P[tail, p0:p0+k] * z   (see DESIGN.md)
      if (threadIdx.x == 0) {
        z[k] = 1.0;
        for (int i = k - 1; i >= 0; i--) {
          double acc = 0.0;
          if (!skipped[i]) for (int j = i + 1; j <= k; j++) acc += A[j][i] * z[j];
          z[i] = -acc;
        }
      }
      __syncthreads();
      ArgMax am{-1.0, 0x7fffffff};
      // sub-diagonal rows inside the block come first (index = position in the sub-column)
      for (int r = k + 1 + threadIdx.x; r < w; r += blockDim.x) am = am_better(am, ArgMax{fabs(A[r][k]), r - (k + 1)});
      for (int r = p0 + w + threadIdx.x; r < m; r += blockDim.x) {
        double v = 0.0;
        for (int j = 0; j <= k; j++) v += P[(long long)(p0 + j) * ld + r] * z[j];
        vscratch[r] = v;
        am = am_better(am, ArgMax{fabs(v), r - (p0 + k + 1)});
      }
      am = block_argmax(am, sh_am);
      if (threadIdx.x == 0) {
        int t = am.i + 1;                                // position in the sub-column
        int sublen = collen - 1;
        double v;
        if (t < sublen) {
          int r = p0 + k + 1 + t;                        // row inside the panel
          v = (r < p0 + w) ? A[r - p0][k] : vscratch[r];
        } else if (k + 1 < w) {
          v = A[k + 1][k + 1];
        } else if (p0 + w < n) {
          // diagonal of the next panel's first column as the reference would hold it now:
          // updated by the columns 0..k-1 of this panel (column k not applied yet)
          int r = p0 + w;
          double u[NB];
          double x = P[(long long)r * ld + r];
          for (int j = 0; j < k; j++) {
            double uj = P[(long long)(p0 + j) * ld + r];
            for (int i = 0; i < j; i++) if (!skipped[i]) uj -= u[i] * A[j][i];
            u[j] = uj;
            if (!skipped[j]) x -= uj * uj / dloc[j];
          }
          v = x;
        } else {
          v = (gk + 1 < mtot) ? diagX[gk + 1] : 0.0;
        }
        double ubk = fabs(v) / maxu;
        if (xkk < ubk) { flag[gk] = 2; sval[gk] = ubk - xkk; xkk = ubk; }
        s_x = xkk;
      }
      __syncthreads();
      xkk = s_x;
      __syncthreads();
    }
    if (skip) {
      if (threadIdx.x == 0) { d[gk] = 0.0; flag[gk] = 1; sval[gk] = xkk; skipped[k] = 1; dloc[k] = 0.0; }
      __syncthreads();
      continue;
    }
    // rank-1 update inside the block with the undivided column
    for (int idx = threadIdx.x; idx < (w - k - 1) * (w - k - 1); idx += blockDim.x) {
      int r = k + 1 + idx % (w - k - 1), c = k + 1 + idx / (w - k - 1);
      if (r >= c) A[r][c] -= (A[c][k] / xkk) * A[r][k];
    }
    __syncthreads();
    for (int r = k + 1 + threadIdx.x; r < w; r += blockDim.x) A[r][k] /= xkk;
    if (threadIdx.x == 0) { d[gk] = xkk; dloc[k] = xkk; A[k][k] = 1.0; }
    __syncthreads();
  }
  // write L11 back; skipped columns: zero below the diagonal (excluded from everything later)
  for (int idx = threadIdx.x; idx < w * w; idx += blockDim.x) {
    int r = idx % w, c = idx / w;
    if (r >= c) P[(long long)(p0 + c) * ld + p0 + r] = (skipped[c] && r > c) ? 0.0 : A[r][c];
  }
}

// trsm kernel: rows below the diagonal block:  L21 = A21 * L11^-T * D^-1  (one thread per row)
__global__ void __launch_bounds__(128)
trsm_kernel(Sn s, int p0, int w, double *rect, const double *d) {
  __shared__ double L11[NB][NB + 1];
  __shared__ double dl[NB];
  double *P = rect + s.poff;
  const int ld = s.m;
  for (int idx = threadIdx.x; idx < w * w; idx += blockDim.x) {
    int r = idx % w, c = idx / w;
    L11[r][c] = (r > c) ? P[(long long)(p0 + c) * ld + p0 + r] : 0.0;
  }
  if (threadIdx.x < w) dl[threadIdx.x] = d[s.first + p0 + threadIdx.x];
  __syncthreads();
  int r = p0 + w + blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= s.m) return;
  double a[NB];
#pragma unroll
  for (int j = 0; j < NB; j++) a[j] = (j < w) ? P[(long long)(p0 + j) * ld + r] : 0.0;
#pragma unroll
  for (int j = 0; j < NB; j++) {
    if (j < w) {
      double dj = dl[j];
      double xj = a[j];                                   // undivided, fully updated
      if (dj > 0.0) {
#pragma unroll
        for (int j2 = j + 1; j2 < NB; j2++) if (j2 < w) a[j2] -= xj * L11[j2][j];
        a[j] = xj / dj;
      } else a[j] = 0.0;                                  // skipped pivot: column excluded
    }
  }
#pragma unroll
  for (int j = 0; j < NB; j++) if (j < w) P[(long long)(p0 + j) * ld + r] = a[j];
}

// trailing update:  C[r,c] -= sum_j L21[r,j] d_j L21[c,j]   (r >= c), 64x64 tiles, 4x4 per thread
__global__ void __launch_bounds__(256)
trail_kernel(Sn s, int p0, int w, double *rect, const double *d) {
  const int base = p0 + w;
  const int r0 = base + blockIdx.x * 64, c0 = base + blockIdx.y * 64;
  if (r0 + 63 < c0 || c0 >= s.n || r0 >= s.m) return;     // tile entirely above the diagonal / outside
  __shared__ double As[NB][64 + 1], Bs[NB][64 + 1];
  double *P = rect + s.poff;
  const int ld = s.m;
  for (int idx = threadIdx.x; idx < 64 * w; idx += blockDim.x) {
    int i = idx % 64, j = idx / 64;
    int r = r0 + i, c = c0 + i;
    As[j][i] = (r < s.m) ? P[(long long)(p0 + j) * ld + r] : 0.0;
    Bs[j][i] = (c < s.n) ? P[(long long)(p0 + j) * ld + c] * d[s.first + p0 + j] : 0.0;
  }
  __syncthreads();
  const int tx = threadIdx.x % 16, ty = threadIdx.x / 16;
  double acc[4][4] = {};
  for (int j = 0; j < w; j++) {
    double av[4], bv[4];
#pragma unroll
    for (int i = 0; i < 4; i++) { av[i] = As[j][tx + 16 * i]; bv[i] = Bs[j][ty + 16 * i]; }
#pragma unroll
    for (int i = 0; i < 4; i++)
#pragma unroll
      for (int q = 0; q < 4; q++) acc[i][q] += av[i] * bv[q];
  }
#pragma unroll
  for (int q = 0; q < 4; q++) {
    int c = c0 + ty + 16 * q;
    if (c >= s.n) continue;
#pragma unroll
    for (int i = 0; i < 4; i++) {
      int r = r0 + tx + 16 * i;
      if (r < s.m && r >= c) P[(long long)c * ld + r] -= acc[i][q];
    }
  }
}

// ======================================================================= layout conversion
__global__ void rect_to_csc_kernel(const Sn *sn, const int *snode, const long long *Ljc,
                                   const double *rect, const int *flag, double *Lpr) {
  int j = blockIdx.x;
  Sn s = sn[snode[j]];
  int c = j - s.first;
  const double *col = rect + s.poff + (long long)c * s.m;
  double *out = Lpr + Ljc[j];
  bool sk = flag && flag[j] == 1;
  for (int t = c + threadIdx.x; t < s.m; t += blockDim.x)
    out[t - c] = (t == c) ? 1.0 : (sk ? 0.0 : col[t]);
}
__global__ void csc_to_rect_kernel(const Sn *sn, const int *snode, const long long *Ljc,
                                   const double *Lpr, double *rect) {
  int j = blockIdx.x;
  Sn s = sn[snode[j]];
  int c = j - s.first;
  double *col = rect + s.poff + (long long)c * s.m;
  const double *in = Lpr + Ljc[j];
  for (int t = threadIdx.x; t < s.m; t += blockDim.x) col[t] = (t >= c) ? in[t - c] : 0.0;
}

// ======================================================================= solves
// Forward: one CTA per (supernode of the level, rhs).  y has length m per rhs, already = b(perm).
__global__ void __launch_bounds__(512)
fwsolve_kernel(const int *list, const Sn *sn, const int *pull_ptr, const int *pull_src, const int *pull_K,
               const unsigned char *kmask, const double *rect, double *y, int m, int solve, double *cvec, long long ctot) {
  extern __shared__ double sm[];             // s[n]
  Sn sj = sn[list[blockIdx.x]];
  double *yy = y + (long long)blockIdx.y * m;
  double *cv = cvec + (long long)blockIdx.y * ctot;
  const int n = sj.n;
  double *s = sm;
  for (int c = threadIdx.x; c < n; c += blockDim.x) s[c] = yy[sj.first + c];
  __syncthreads();
  // pull the contributions c_K = L21_K y_K of the descendants, in list order:  s[col] -= c_K[row]
  // (thread c owns s[c]: its contributions are listed in the plan, in descendant order)
  for (int c = threadIdx.x; c < n; c += blockDim.x) {
    double acc = 0.0;
    for (int q = pull_ptr[sj.first + c]; q < pull_ptr[sj.first + c + 1]; q++)
      if (!kmask || kmask[pull_K[q]]) acc += cv[pull_src[q]];
    s[c] -= acc;
  }
  __syncthreads();
  // dense unit-lower solve of the n x n diagonal block, 32 columns at a time (solve = 0: pull only, used by the
  // sharded forward pass to collect the contributions of a rank's subtrees in the replicated top rows)
  const double *P = rect + sj.poff;
  const int ld = sj.m;
  for (int k0 = 0; solve && k0 < n; k0 += 32) {
    int w = min(32, n - k0);
    if (threadIdx.x < 32) {
      int lane = threadIdx.x;
      double v = (lane < w) ? s[k0 + lane] : 0.0;
      double lr[32];                                    // row `lane` of the diagonal block: all loads in flight before the chain starts
#pragma unroll
      for (int k = 0; k < 32; k++) lr[k] = (k < w && lane > k && lane < w) ? P[(long long)(k0 + k) * ld + k0 + lane] : 0.0;
#pragma unroll
      for (int k = 0; k < 32; k++) {
        double yk = __shfl_sync(0xffffffffu, v, k);
        v -= lr[k] * yk;
      }
      if (lane < w) s[k0 + lane] = v;
    }
    __syncthreads();
    for (int r = k0 + w + threadIdx.x; r < n; r += blockDim.x) {
      double acc = 0.0;
      for (int k = 0; k < w; k++) acc += P[(long long)(k0 + k) * ld + r] * s[k0 + k];
      s[r] -= acc;
    }
    __syncthreads();
  }
  for (int c = threadIdx.x; c < n; c += blockDim.x) yy[sj.first + c] = s[c];
  // this supernode's own contribution to its ancestors: c_J = L21 y_J
  const int mk = sj.m - n;
  if (solve && mk > 0) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = blockDim.x >> 5;
    double *cj = cv + sj.cvoff;
    if (mk >= 256) {                                      // long tails: one thread per row (coalesced over rows)
      for (int t = threadIdx.x; t < mk; t += blockDim.x) {
        double acc = 0.0;
        for (int k = 0; k < n; k++) acc += P[(long long)k * ld + n + t] * s[k];
        cj[t] = acc;
      }
    } else {                                              // short tails: 32 rows per warp pass, columns split over warps
      __syncthreads();
      double *part = sm + n;                              // [nw][mk] partial sums (the launcher sizes shared memory for it)
      for (int t0 = 0; t0 < mk; t0 += 32) {
        const int t = t0 + lane;
        double acc = 0.0;
        if (t < mk) for (int k = warp; k < n; k += nw) acc += P[(long long)k * ld + n + t] * s[k];
        if (t < mk) part[warp * mk + t] = acc;
      }
      __syncthreads();
      for (int t = threadIdx.x; t < mk; t += blockDim.x) {
        double acc = 0.0;
        for (int w = 0; w < nw; w++) acc += part[w * mk + t];
        cj[t] = acc;
      }
    }
  }
}

// Backward: z = L'^-1 b in permuted order, levels descending.
__global__ void __launch_bounds__(512)
bwsolve_kernel(const int *list, const Sn *sn, const int *lindx, const double *rect, double *z, int m) {
  extern __shared__ double sm[];
  Sn sj = sn[list[blockIdx.x]];
  double *zz = z + (long long)blockIdx.y * m;
  const int n = sj.n, ld = sj.m;
  const double *P = rect + sj.poff;
  const int *rows = lindx + sj.lindx;
  double *s = sm;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = blockDim.x >> 5;
  // s[c] = b[c] - sum_{t>=n} L[t,c] * z[rows[t]]
  for (int c = warp; c < n; c += nw) {
    const double *col = P + (long long)c * ld;
    double acc = 0.0;
    for (int t = n + lane; t < sj.m; t += 32) acc += col[t] * zz[rows[t]];
    for (int o = 16; o > 0; o >>= 1) acc += __shfl_down_sync(0xffffffffu, acc, o);
    if (lane == 0) s[c] = zz[sj.first + c] - acc;
  }
  __syncthreads();
  for (int k1 = n; k1 > 0; k1 -= 32) {
    int k0 = max(0, k1 - 32), w = k1 - k0;
    if (threadIdx.x < 32) {
      double v = (lane < w) ? s[k0 + lane] : 0.0;
      double lc[32];                                    // column `lane` of the diagonal block, fetched before the chain starts
#pragma unroll
      for (int k = 0; k < 32; k++) lc[k] = (k < w && lane < k) ? P[(long long)(k0 + lane) * ld + k0 + k] : 0.0;
#pragma unroll
      for (int k = 31; k >= 0; k--) {
        double zk = __shfl_sync(0xffffffffu, v, k);
        // z_c -= L[k, c] * z_k for c < k
        v -= lc[k] * zk;
      }
      if (lane < w) s[k0 + lane] = v;
    }
    __syncthreads();
    for (int c = threadIdx.x; c < k0; c += blockDim.x) {
      const double *col = P + (long long)c * ld + k0;
      double acc = 0.0;
      for (int k = 0; k < w; k++) acc += col[k] * s[k0 + k];
      s[c] -= acc;
    }
    __syncthreads();
  }
  for (int c = threadIdx.x; c < n; c += blockDim.x) zz[sj.first + c] = s[c];
}

// w(i,col) /= d_i with deninfac's repair of skipped pivots (deninfac.m:88-93): a skipped pivot
// (flag==1) whose d is <= max(abstol, canceltol*absd(perm_i)) (= lb_i) is replaced by 1.
__global__ void scale_by_d_kernel(int m, int nrhs, const double *d, const int *flag, const double *lb, double *w) {
  long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i >= (long long)m * nrhs) return;
  int k = (int)(i % m);
  double dk = d[k];
  if (flag && flag[k] == 1 && dk <= lb[k]) dk = 1.0;
  w[i] /= dk;
}

// ssqr = sum_i w_i^2 d_i with deninfac's repaired pivots (one block: m is at most a few thousand)
__global__ void __launch_bounds__(1024) ssqr_kernel(int m, const double *d, const int *flag, const double *lb, const double *w, double *out) {
  __shared__ double sh[32];
  double a = 0.0;
  for (int k = threadIdx.x; k < m; k += blockDim.x) {
    double dk = d[k];
    if (flag && flag[k] == 1 && dk <= lb[k]) dk = 1.0;
    a += w[k] * w[k] * dk;
  }
  for (int o = 16; o > 0; o >>= 1) a += __shfl_down_sync(0xffffffffu, a, o);
  if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = a;
  __syncthreads();
  if (threadIdx.x == 0) { double t = 0.0; for (int i = 0; i < 32; i++) t += sh[i]; *out = t; }
}

__global__ void gather_perm_kernel(int m, int nrhs, const int *perm, const double *b, double *y) {
  long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i >= (long long)m * nrhs) return;
  int k = (int)(i % m); long long col = i / m;
  y[i] = b[col * m + perm[k]];
}
__global__ void scatter_perm_kernel(int m, int nrhs, const int *perm, const double *z, double *y) {
  long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i >= (long long)m * nrhs) return;
  int k = (int)(i % m); long long col = i / m;
  y[col * m + perm[k]] = z[i];
}

}  // namespace sb

// =========================================================================== host side
using namespace sb;

// one CTA factors the whole panel: narrow supernodes, or any panel that fits the CTA's shared memory
static inline bool sn_is_small(const sb200_chol_plan *pl, const Sn &S) {
  return S.n <= SMALL_N || (size_t)S.m * S.n <= pl->small_cap;
}
static inline size_t small_shm(const sb200_chol_plan *pl, const std::vector<int> &list) {
  size_t need = 0;
  for (int s : list) { const size_t e = (size_t)pl->sn[s].m * pl->sn[s].n; if (e <= pl->small_cap) need = std::max(need, e); }
  return need * sizeof(double);
}
static inline int schur_tiles(const sb200_chol_plan *pl, const std::vector<int> &list) {
  int mx = 0;
  for (int s : list) { const int nt = (pl->sn[s].m - pl->sn[s].n + 63) / 64; mx = std::max(mx, nt * (nt + 1) / 2); }
  return mx;
}
static int launch_factor_small(sb200_chol_plan *pl, const std::vector<int> &list, const int *list_dev, sb200_chol_pars pars, double *rect,
                               double *d, int *flag, double *sval) {
  if (list.empty()) return 0;
  const size_t shm = small_shm(pl, list);
  static size_t attr = 0;
  if (shm > attr) { SB_CUDA(cudaFuncSetAttribute(factor_small_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(pl->small_cap * sizeof(double)))); attr = pl->small_cap * sizeof(double); }
  factor_small_kernel<<<(unsigned)list.size(), 512, shm, ctx().stream>>>(list_dev, pl->d_sn.p, rect, d, pl->d_lb.p, pl->d_scal.p, pars.maxu, flag, sval,
                                                                          pl->d_diagX.p, pl->m, (int)pl->small_cap);
  SB_LAUNCH_CHECK_N("factor_small_kernel");
  return 0;
}
static int launch_schur(sb200_chol_plan *pl, const std::vector<int> &list, const int *list_dev, const double *rect, const double *d) {
  const int nt = schur_tiles(pl, list);
  if (list.empty() || nt == 0) return 0;
  schur_kernel<<<dim3((unsigned)list.size(), (unsigned)nt), 256, 0, ctx().stream>>>(list_dev, pl->d_sn.p, rect, d, pl->d_U.p);
  SB_LAUNCH_CHECK_N("schur_kernel");
  return 0;
}
// shared memory of a forward-solve CTA: the supernode's part of y + the per-warp partial sums of its contribution
static inline size_t fw_shm(const sb200_chol_plan *pl) {
  size_t need = 0;
  for (auto &S : pl->sn) { const int mk = S.m - S.n; need = std::max(need, (size_t)S.n + (mk < 256 ? (size_t)16 * mk : 0)); }
  return need * sizeof(double);
}
static int ensure_cvec(sb200_chol_plan *pl, int nrhs) {
  if (pl->cvec_nrhs >= nrhs && pl->d_cvec.p) return 0;
  SB_CHECK(!ctx().capturing, "solve: the contribution workspace must be sized before graph capture (run one solve first)");
  SB_TRY(pl->d_cvec.alloc((size_t)std::max<long long>(pl->ctot, 1) * nrhs));
  pl->cvec_nrhs = nrhs;
  return 0;
}

static int build_plan(sb200_chol_plan *pl, sb_idx m64, sb_idx nsuper64, const sb_idx *xsuper,
                      const sb_idx *Ljc, const sb_idx *Lir, const sb_idx *perm,
                      const sb_idx *Xjc, const sb_idx *Xir) {
  SB_CHECK(m64 >= 0 && m64 < 2147483647LL, "blkchol: m out of range");
  const int m = (int)m64, nsuper = (int)nsuper64;
  pl->m = m; pl->nsuper = nsuper;
  pl->nnzL = Ljc[m];
  SB_CHECK(nsuper >= 0 && nsuper <= m, "blkchol: Size L.xsuper mismatch.");
  SB_CHECK(xsuper[0] == 0 && xsuper[nsuper] == m, "blkchol: L.xsuper must span 1..m+1");
  pl->sn.resize(nsuper);
  pl->snode.assign(m, 0);
  std::vector<int> lindx;
  long long poff = 0;
  for (int s = 0; s < nsuper; s++) {
    Sn &S = pl->sn[s];
    S.first = (int)xsuper[s];
    S.n = (int)(xsuper[s + 1] - xsuper[s]);
    SB_CHECK(S.n > 0, "blkchol: empty supernode %d", s);
    S.m = (int)(Ljc[S.first + 1] - Ljc[S.first]);
    SB_CHECK(S.m >= S.n, "blkchol: supernode %d shorter than its width", s);
    S.lindx = (int)lindx.size();
    S.poff = poff;
    S.coff = Ljc[S.first];
    poff += (long long)S.m * S.n;
    poff = (poff + 1) & ~1LL;                 // panels start on 16-byte boundaries: they move through the TMA unit as bulk copies
    for (int t = 0; t < S.m; t++) {
      sb_idx r = Lir[Ljc[S.first] + t];
      SB_CHECK(r >= 0 && r < m, "blkchol: L.L row index out of range");
      if (t < S.n) SB_CHECK(r == S.first + t, "blkchol: L.L is not a supernodal pattern (column %d)", S.first);
      lindx.push_back((int)r);
    }
    for (int c = 0; c < S.n; c++) {
      pl->snode[S.first + c] = s;
      SB_CHECK(Ljc[S.first + c + 1] - Ljc[S.first + c] == S.m - c, "blkchol: column %d breaks the nested supernode pattern", S.first + c);
    }
    pl->max_sn_n = std::max(pl->max_sn_n, S.n);
    pl->max_sn_m = std::max(pl->max_sn_m, S.m);
  }
  pl->rect = poff;
  // contribution blocks (Schur complement of every supernode on its rows below the diagonal block, and its share of
  // the forward solve): offsets
  {
    long long uo = 0, co = 0;
    for (int s = 0; s < nsuper; s++) {
      Sn &S = pl->sn[s];
      const long long mk = S.m - S.n;
      S.uoff = uo; S.cvoff = (int)co; S.pad_ = 0;
      uo += mk * mk; co += mk;
      pl->max_mk = std::max(pl->max_mk, (int)mk);
    }
    SB_CHECK(co < 2147483647LL, "blkchol: factor too large for 32-bit contribution offsets");
    pl->utot = uo; pl->ctot = co;
    pl->small_cap = 27000;                               // 216 KB of shared memory for a factor CTA's panel
  }
  // update pairs
  std::vector<std::vector<Pair>> byJ(nsuper);
  std::vector<int> rel;
  pl->level_of.assign(nsuper, 0);
  for (int K = 0; K < nsuper; K++) {
    const Sn &SK = pl->sn[K];
    const int *rk = lindx.data() + SK.lindx;
    int t = SK.n;
    while (t < SK.m) {
      int J = pl->snode[rk[t]];
      SB_CHECK(J > K, "blkchol: row structure of supernode %d is not ascending", K);
      int t0 = t;
      while (t < SK.m && pl->snode[rk[t]] == J) t++;
      Pair p; p.K = K; p.J = J; p.koff = t0; p.mk = SK.m - t0; p.ncolup = t - t0; p.rel = (int)rel.size();
      const Sn &SJ = pl->sn[J];
      const int *rj = lindx.data() + SJ.lindx;
      int pos = 0;
      for (int tt = t0; tt < SK.m; tt++) {
        while (pos < SJ.m && rj[pos] < rk[tt]) pos++;
        SB_CHECK(pos < SJ.m && rj[pos] == rk[tt], "blkchol: structure of supernode %d not contained in ancestor %d", K, J);
        rel.push_back(pos);
      }
      byJ[J].push_back(p);
      pl->level_of[J] = std::max(pl->level_of[J], pl->level_of[K] + 1);
    }
  }
  std::vector<Pair> pairs;
  pl->pair_beg.assign(nsuper + 1, 0);
  for (int J = 0; J < nsuper; J++) {
    pl->pair_beg[J] = (int)pairs.size();
    for (auto &p : byJ[J]) pairs.push_back(p);
  }
  pl->pair_beg[nsuper] = (int)pairs.size();
  // gather lists (counting sort by target keeps the descendant order inside each target)
  {
    std::vector<int> pptr(m + 1, 0);
    for (auto &p : pairs) for (int t = 0; t < p.ncolup; t++) pptr[pl->sn[p.J].first + rel[p.rel + t] + 1]++;
    for (int c = 0; c < m; c++) pptr[c + 1] += pptr[c];
    std::vector<int> psrc((size_t)std::max(pptr[m], 1)), pK((size_t)std::max(pptr[m], 1)), fill(pptr.begin(), pptr.end() - 1);
    for (auto &p : pairs) {
      const Sn &SK = pl->sn[p.K];
      for (int t = 0; t < p.ncolup; t++) { const int q = fill[pl->sn[p.J].first + rel[p.rel + t]]++; psrc[q] = SK.cvoff + (p.koff - SK.n) + t; pK[q] = p.K; }
    }
    SB_TRY(pl->d_pull_ptr.upload(pptr)); SB_TRY(pl->d_pull_src.upload(psrc)); SB_TRY(pl->d_pull_K.upload(pK));
    long long items = 0;
    for (auto &p : pairs) items += (long long)p.ncolup * p.mk - (long long)p.ncolup * (p.ncolup - 1) / 2;
    pl->upd_lists = !pairs.empty() && items < ((long long)1 << 28) && pl->rect < ((long long)1 << 30);
    if (pl->upd_lists) {
      std::vector<int> uptr((size_t)pl->rect + 1, 0);
      for (auto &p : pairs) {
        const Sn &SJ = pl->sn[p.J];
        for (int t2 = 0; t2 < p.ncolup; t2++)
          for (int t1 = t2; t1 < p.mk; t1++) uptr[SJ.poff + rel[p.rel + t1] + (long long)rel[p.rel + t2] * SJ.m + 1]++;
      }
      for (long long e = 0; e < pl->rect; e++) uptr[e + 1] += uptr[e];
      std::vector<long long> usrc((size_t)std::max<long long>(items, 1));
      std::vector<int> uK((size_t)std::max<long long>(items, 1)), ufill(uptr.begin(), uptr.end() - 1);
      for (auto &p : pairs) {
        const Sn &SJ = pl->sn[p.J], &SK = pl->sn[p.K];
        const long long mk = SK.m - SK.n, u0 = p.koff - SK.n;
        for (int t2 = 0; t2 < p.ncolup; t2++)
          for (int t1 = t2; t1 < p.mk; t1++) {
            const int q = ufill[SJ.poff + rel[p.rel + t1] + (long long)rel[p.rel + t2] * SJ.m]++;
            usrc[q] = SK.uoff + (u0 + t1) + (u0 + t2) * mk; uK[q] = p.K;
          }
      }
      SB_TRY(pl->d_upd_ptr.upload(uptr)); SB_TRY(pl->d_upd_src.upload(usrc)); SB_TRY(pl->d_upd_K.upload(uK));
    }
  }
  int nlev = 0;
  for (int s = 0; s < nsuper; s++) nlev = std::max(nlev, pl->level_of[s] + 1);
  pl->nlevels = nlev;
  pl->level_small.assign(nlev, {}); pl->level_big.assign(nlev, {}); pl->level_tiles.assign(nlev, {});
  pl->level_all.assign(nlev, {});
  for (int s = 0; s < nsuper; s++) {
    int lv = pl->level_of[s];
    (sn_is_small(pl, pl->sn[s]) ? pl->level_small : pl->level_big)[lv].push_back(s);
    pl->level_all[lv].push_back(s);
    if (pl->pair_beg[s + 1] > pl->pair_beg[s]) {
      const Sn &S = pl->sn[s];
      for (int c0 = 0; c0 < S.n; c0 += UT_C)
        for (int r0 = (c0 / UT_R) * UT_R; r0 < S.m; r0 += UT_R) pl->level_tiles[lv].push_back(UTile{s, r0, c0});
    }
  }
  std::vector<int> small_list, all_list; std::vector<UTile> tiles;
  for (int lv = 0; lv < nlev; lv++) {
    pl->level_small_off.push_back((int)small_list.size());
    pl->level_tile_off.push_back((int)tiles.size());
    pl->level_all_off.push_back((int)all_list.size());
    for (int s : pl->level_small[lv]) small_list.push_back(s);
    for (int s : pl->level_all[lv]) all_list.push_back(s);
    for (auto &t : pl->level_tiles[lv]) tiles.push_back(t);
  }
  std::vector<int> perm32, Xjc32, Xir32;
  SB_TRY(to_i32(perm, m, perm32, "L.perm"));
  SB_TRY(to_i32(Xjc, m + 1, Xjc32, "X.jc"));
  SB_TRY(to_i32(Xir, (size_t)Xjc[m], Xir32, "X.ir"));
  for (int i = 0; i < m; i++) SB_CHECK(perm32[i] < m, "blkchol: perm out of range");
  std::vector<long long> Ljc64(Ljc, Ljc + m + 1);
  SB_TRY(pl->d_sn.upload(pl->sn));
  SB_TRY(pl->d_pairs.upload(pairs));
  SB_TRY(pl->d_pair_beg.upload(pl->pair_beg));
  SB_TRY(pl->d_rel.upload(rel));
  SB_TRY(pl->d_lindx.upload(lindx));
  SB_TRY(pl->d_snode.upload(pl->snode));
  SB_TRY(pl->d_perm.upload(perm32));
  SB_TRY(pl->d_Xjc.upload(Xjc32));
  SB_TRY(pl->d_Xir.upload(Xir32));
  SB_TRY(pl->d_level_list.upload(small_list));
  SB_TRY(pl->d_level_all.upload(all_list));
  SB_TRY(pl->d_tiles.upload(tiles));
  SB_TRY(pl->d_Ljc.upload(Ljc64));
  SB_TRY(pl->d_diagX.alloc(m));
  SB_TRY(pl->d_lb.alloc(m));
  SB_TRY(pl->d_scal.alloc(8));
  SB_TRY(pl->d_vscratch.alloc(std::max(pl->max_sn_m, 1)));
  if (nsuper > 1) SB_TRY(pl->d_U.alloc((size_t)std::max<long long>(pl->utot, 1)));
  pl->dense_fast = (nsuper == 1 && m >= 1 && pl->sn[0].m == m && pl->sn[0].n == m &&
                    (size_t)m * 8 + 8 * 2 * 1024 * 8 + 8192 <= 200 * 1024);   // shared memory of the dataflow solves
  if (pl->dense_fast) SB_TRY(dense_factor_prepare(pl));
  SB_CUDA(cudaStreamSynchronize(ctx().stream));       // host vectors go out of scope
  return 0;
}

extern "C" {

int sb200_chol_plan_create(sb200_chol_plan **plan, sb_idx m, sb_idx nsuper, const sb_idx *xsuper,
                           const sb_idx *Ljc, const sb_idx *Lir, const sb_idx *perm,
                           const sb_idx *Xjc, const sb_idx *Xir) {
  SB_TRY(ensure_init());
  sb200_chol_plan *pl = new sb200_chol_plan();
  int rc = build_plan(pl, m, nsuper, xsuper, Ljc, Lir, perm, Xjc, Xir);
  if (rc) { delete pl; return rc; }
  *plan = pl;
  return 0;
}
void sb200_chol_plan_destroy(sb200_chol_plan *plan) { delete plan; }
sb_idx sb200_chol_plan_nnzL(const sb200_chol_plan *plan) { return plan->nnzL; }
const double *sb200_chol_plan_lb_dev(const sb200_chol_plan *plan) { return plan->d_lb.p; }
sb_idx sb200_chol_plan_rect_size(const sb200_chol_plan *plan) { return plan->rect; }

static void launch_bounds_cb(sb200_chol_plan *pl, const double *absd, sb200_chol_pars pars) {
  bounds_kernel<<<1, 1024, 0, ctx().stream>>>(pl->m, pl->d_diagX.p, absd, pl->d_perm.p, pars.abstol, pars.canceltol,
                                              pars.maxu, pl->d_lb.p, pl->d_scal.p);
  ctx().launches++;
  if (ctx().profiling) prof_mark("bounds_kernel");
}

int sb200_blkchol_dev(sb200_chol_plan *pl, const double *Xpr, const double *absd,
                      sb200_chol_pars pars, double *rect, double *d, int *flag, double *sval) {
  SB_TRY(ensure_init());
  cudaStream_t st = ctx().stream;
  const int m = pl->m;
  if (m == 0) return 0;
  SB_CUDA(cudaMemsetAsync(flag, 0, sizeof(int) * m, st));
  SB_CUDA(cudaMemsetAsync(sval, 0, sizeof(double) * m, st));
  if (pl->dense_fast) return dense_factor(pl, Xpr, absd, pars, rect, d, flag, sval, launch_bounds_cb);
  permuteP_kernel<<<m, 256, 0, st>>>(pl->d_sn.p, pl->d_snode.p, pl->d_lindx.p, pl->d_perm.p,
                                      pl->d_Xjc.p, pl->d_Xir.p, Xpr, rect, pl->d_diagX.p);
  SB_LAUNCH_CHECK_N("permuteP_kernel");
  bounds_kernel<<<1, 1024, 0, st>>>(m, pl->d_diagX.p, absd, pl->d_perm.p, pars.abstol, pars.canceltol,
                                     pars.maxu, pl->d_lb.p, pl->d_scal.p);
  SB_LAUNCH_CHECK_N("bounds_kernel");
  for (int lv = 0; lv < pl->nlevels; lv++) {
    int ntile = (int)pl->level_tiles[lv].size();
    if (ntile) {
      if (pl->upd_lists)
        update_gather_kernel<<<ntile, 256, 0, st>>>(pl->d_tiles.p + pl->level_tile_off[lv], pl->d_sn.p, pl->d_upd_ptr.p, pl->d_upd_src.p,
                                                    pl->d_upd_K.p, nullptr, pl->d_U.p, rect);
      else
        update_kernel<<<ntile, 256, 0, st>>>(pl->d_tiles.p + pl->level_tile_off[lv], pl->d_sn.p, pl->d_pairs.p,
                                              pl->d_pair_beg.p, pl->d_rel.p, pl->d_U.p, rect);
      SB_LAUNCH_CHECK_N("update_kernel");
    }
    SB_TRY(launch_factor_small(pl, pl->level_small[lv], pl->d_level_list.p + pl->level_small_off[lv], pars, rect, d, flag, sval));
    for (int s : pl->level_big[lv]) {
      const Sn &S = pl->sn[s];
      for (int p0 = 0; p0 < S.n; p0 += NB) {
        int w = std::min(NB, S.n - p0);
        diag_kernel<<<1, 256, 0, st>>>(S, p0, w, rect, d, pl->d_lb.p, pl->d_scal.p, pars.maxu, flag, sval,
                                        pl->d_diagX.p, m, pl->d_vscratch.p);
        SB_LAUNCH_CHECK_N("diag_kernel");
        int nrow = S.m - (p0 + w);
        if (nrow > 0) {
          trsm_kernel<<<(nrow + 127) / 128, 128, 0, st>>>(S, p0, w, rect, d);
          SB_LAUNCH_CHECK_N("trsm_kernel");
          int ncol = S.n - (p0 + w);
          if (ncol > 0) {
            dim3 g((nrow + 63) / 64, (ncol + 63) / 64);
            trail_kernel<<<g, 256, 0, st>>>(S, p0, w, rect, d);
            SB_LAUNCH_CHECK_N("trail_kernel");
          }
        }
      }
    }
    if (lv + 1 < pl->nlevels) SB_TRY(launch_schur(pl, pl->level_all[lv], pl->d_level_all.p + pl->level_all_off[lv], rect, d));
  }
  return 0;
}

int sb200_chol_rect_to_csc_dev(sb200_chol_plan *pl, const double *rect, const int *flag, double *Lpr) {
  SB_TRY(ensure_init());
  if (pl->m == 0) return 0;
  rect_to_csc_kernel<<<pl->m, 128, 0, ctx().stream>>>(pl->d_sn.p, pl->d_snode.p, pl->d_Ljc.p, rect, flag, Lpr);
  SB_LAUNCH_CHECK_N("rect_to_csc_kernel");
  return 0;
}
int sb200_chol_csc_to_rect_dev(sb200_chol_plan *pl, const double *Lpr, double *rect) {
  SB_TRY(ensure_init());
  if (pl->m == 0) return 0;
  csc_to_rect_kernel<<<pl->m, 128, 0, ctx().stream>>>(pl->d_sn.p, pl->d_snode.p, pl->d_Ljc.p, Lpr, rect);
  SB_LAUNCH_CHECK_N("csc_to_rect_kernel");
  return 0;
}

int sb200_fwblkslv_dev(sb200_chol_plan *pl, const double *rect, const double *b, double *y, sb_idx nrhs) {
  SB_TRY(ensure_init());
  cudaStream_t st = ctx().stream;
  const int m = pl->m;
  if (m == 0 || nrhs == 0) return 0;
  if (pl->dense_fast) return dense_fwsolve(pl, rect, b, y, (int)nrhs, nullptr, nullptr);
  long long tot = (long long)m * nrhs;
  gather_perm_kernel<<<(unsigned)((tot + 255) / 256), 256, 0, st>>>(m, (int)nrhs, pl->d_perm.p, b, y);
  SB_LAUNCH_CHECK_N("gather_perm_kernel");
  size_t shm = fw_shm(pl);
  SB_CHECK(shm <= 200 * 1024, "fwblkslv: supernode wider than the shared-memory solve supports (%d)", pl->max_sn_n);
  if (shm > 48 * 1024) SB_CUDA(cudaFuncSetAttribute(fwsolve_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)shm));
  SB_TRY(ensure_cvec(pl, (int)nrhs));
  for (int lv = 0; lv < pl->nlevels; lv++) {
    dim3 g((unsigned)pl->level_all[lv].size(), (unsigned)nrhs);
    fwsolve_kernel<<<g, 512, shm, st>>>(pl->d_level_all.p + pl->level_all_off[lv], pl->d_sn.p, pl->d_pull_ptr.p, pl->d_pull_src.p,
                                         pl->d_pull_K.p, nullptr, rect, y, m, 1, pl->d_cvec.p, pl->ctot);
    SB_LAUNCH_CHECK_N("fwsolve_kernel");
  }
  return 0;
}

int sb200_bwblkslv_dev(sb200_chol_plan *pl, const double *rect, const double *b, double *y, sb_idx nrhs);
// y = L' \ ((L \ b(perm)) ./ d)  -- the preconditioner application of wrapPcg.m:56-59 for a problem
// without dense columns (fwdpr1/bwdpr1 are identities then, fwdpr1.c:132-135).  w: m*nrhs scratch.
// flag_dev/NULL: when given, skipped pivots get d=1 as deninfac.m:88-93 does (uses the plan's lb
// from the last sb200_blkchol_dev call).
int sb200_ldl_solve_dev(sb200_chol_plan *pl, const double *rect, const double *d, const int *flag,
                        const double *b, double *w, double *y, sb_idx nrhs) {
  return sb200_ldl_solve2_dev(pl, rect, d, flag, b, w, y, nrhs, nullptr);
}
// The same, also returning ssqr = p' (p ./ d) with p = L \ b(perm) (wrapPcg.m:56-58, first right-hand side), computed
// from w = p ./ d as sum w_i^2 d_i with the repaired pivots.
int sb200_ldl_solve2_dev(sb200_chol_plan *pl, const double *rect, const double *d, const int *flag,
                         const double *b, double *w, double *y, sb_idx nrhs, double *ssqr_dev) {
  if (pl->dense_fast) SB_TRY(dense_fwsolve(pl, rect, b, w, (int)nrhs, d, flag));
  else {
    SB_TRY(sb200_fwblkslv_dev(pl, rect, b, w, nrhs));
    long long tot = (long long)pl->m * nrhs;
    if (tot > 0) {
      scale_by_d_kernel<<<(unsigned)((tot + 255) / 256), 256, 0, ctx().stream>>>(pl->m, (int)nrhs, d, flag, pl->d_lb.p, w);
      SB_LAUNCH_CHECK_N("scale_by_d_kernel");
    }
  }
  if (ssqr_dev && pl->m > 0) {
    ssqr_kernel<<<1, 1024, 0, ctx().stream>>>(pl->m, d, flag, pl->d_lb.p, w, ssqr_dev);
    SB_LAUNCH_CHECK_N("ssqr_kernel");
  }
  if (pl->dense_fast) return dense_bwsolve(pl, rect, w, y, (int)nrhs);
  return sb200_bwblkslv_dev(pl, rect, w, y, nrhs);
}

int sb200_bwblkslv_dev(sb200_chol_plan *pl, const double *rect, const double *b, double *y, sb_idx nrhs) {
  SB_TRY(ensure_init());
  cudaStream_t st = ctx().stream;
  const int m = pl->m;
  if (m == 0 || nrhs == 0) return 0;
  if (pl->dense_fast) return dense_bwsolve(pl, rect, b, y, (int)nrhs);
  long long tot = (long long)m * nrhs;
  SB_TRY(pl->d_y.n >= (size_t)tot ? 0 : pl->d_y.alloc((size_t)tot));
  SB_CUDA(cudaMemcpyAsync(pl->d_y.p, b, sizeof(double) * tot, cudaMemcpyDeviceToDevice, st));
  size_t shm = sizeof(double) * (size_t)pl->max_sn_n;
  SB_CHECK(shm <= 200 * 1024, "bwblkslv: supernode wider than the shared-memory solve supports (%d)", pl->max_sn_n);
  if (shm > 48 * 1024) SB_CUDA(cudaFuncSetAttribute(bwsolve_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)shm));
  for (int lv = pl->nlevels - 1; lv >= 0; lv--) {
    dim3 g((unsigned)pl->level_all[lv].size(), (unsigned)nrhs);
    bwsolve_kernel<<<g, 512, shm, st>>>(pl->d_level_all.p + pl->level_all_off[lv], pl->d_sn.p, pl->d_lindx.p,
                                         rect, pl->d_y.p, m);
    SB_LAUNCH_CHECK_N("bwsolve_kernel");
  }
  scatter_perm_kernel<<<(unsigned)((tot + 255) / 256), 256, 0, st>>>(m, (int)nrhs, pl->d_perm.p, pl->d_y.p, y);
  SB_LAUNCH_CHECK_N("scatter_perm_kernel");
  return 0;
}


// ======================================================================= subtree sharding (multi-GPU, SURVEY 8e)
// Supernodes are postordered, so any suffix [t0, nsuper) is closed under "parent of": it is the replicated TOP; the
// supernodes below form a forest whose trees are dealt to the ranks (largest first).  A rank factors its trees, adds
// their Schur contributions into the top panels (which start from the ADA values on rank 0 and from zero elsewhere);
// one all-reduce(sum) of the top panels -- done by the caller between sb200_blkchol_shard_local_dev and
// sb200_blkchol_shard_top_dev -- completes them, and every rank factors the top redundantly.  Solves: forward =
// own trees + pull of their contributions into the top rows, all-reduce of the top segment, top; backward = top, own
// trees; entries of foreign trees are zeroed so that a final all-reduce(sum) assembles the solution.
__global__ void shard_mask_kernel(int m, int nrhs, const int *colmask, double *z) {
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i < (long long)m * nrhs && !colmask[i % m]) z[i] = 0.0;
}
__global__ void shard_scale_kernel(int m, int nrhs, const int *colmask, int top_col0, const double *d, const int *flag, const double *lb, double *w) {
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i >= (long long)m * nrhs) return;
  const int c = (int)(i % m);
  if (!colmask[c] && c < top_col0) { w[i] = 0.0; return; }       // foreign tree; the replicated top is kept on every rank
  double dk = d[c];
  if (flag && flag[c] == 1 && dk <= lb[c]) dk = 1.0;
  w[i] /= dk;
}

int sb200_chol_shard_create(sb200_chol_plan *pl, sb_idx world64, sb_idx rank64) {
  SB_TRY(ensure_init());
  SB_CHECK(!pl->dense_fast, "subtree sharding needs a multi-supernode factor (this one is a single dense supernode)");
  const int world = (int)world64, rank = (int)rank64, ns = pl->nsuper;
  SB_CHECK(world >= 1 && rank >= 0 && rank < world, "shard: rank/world out of range");
  delete pl->shard;
  auto *sh = new sb200_chol_plan::Shard();
  pl->shard = sh;
  sh->world = world; sh->rank = rank;
  // parent of a supernode = supernode of its first off-diagonal row
  std::vector<int> lindx((size_t)0);
  std::vector<Pair> pairs(pl->pair_beg[ns]);
  SB_CUDA(cudaMemcpy(pairs.data(), pl->d_pairs.p, sizeof(Pair) * pairs.size(), cudaMemcpyDeviceToHost));
  std::vector<int> parent(ns, -1);
  for (auto &p : pairs) if (parent[p.K] < 0 || p.J < parent[p.K]) parent[p.K] = p.J;
  std::vector<double> cost(ns, 0.0), sub(ns, 0.0);
  for (int s = 0; s < ns; s++) { cost[s] = (double)pl->sn[s].n * pl->sn[s].m * pl->sn[s].m; sub[s] += cost[s]; if (parent[s] >= 0) sub[parent[s]] += sub[s]; }
  double total = 0.0; for (int s = 0; s < ns; s++) total += cost[s];
  // grow the top from the end until the forest below has enough, small enough trees
  int t0 = ns;
  auto forest_ok = [&](int t) {
    int ntrees = 0; double mx = 0.0;
    for (int s = 0; s < t; s++) if (parent[s] < 0 || parent[s] >= t) { ntrees++; mx = std::max(mx, sub[s]); }
    return ntrees >= 2 * world && mx <= 1.25 * total / world;
  };
  while (t0 > 0 && !forest_ok(t0)) t0--;
  if (t0 == 0) { t0 = ns; while (t0 > 0 && !(([&] { int c = 0; for (int s = 0; s < t0; s++) if (parent[s] < 0 || parent[s] >= t0) c++; return c >= world; })())) t0--; }
  sh->t0 = t0;
  // deal the trees (roots: parent outside the forest) to the ranks, heaviest first
  std::vector<int> roots;
  for (int s = 0; s < t0; s++) if (parent[s] < 0 || parent[s] >= t0) roots.push_back(s);
  std::sort(roots.begin(), roots.end(), [&](int a, int b) { return sub[a] != sub[b] ? sub[a] > sub[b] : a < b; });
  std::vector<double> load(world, 0.0);
  std::vector<int> root_owner(ns, -1);
  for (int r : roots) { int w = (int)(std::min_element(load.begin(), load.end()) - load.begin()); root_owner[r] = w; load[w] += sub[r]; }
  sh->owner.assign(ns, -1);
  for (int s = t0 - 1; s >= 0; s--) sh->owner[s] = (parent[s] < 0 || parent[s] >= t0) ? root_owner[s] : sh->owner[parent[s]];
  // top region of rect / of the column space
  sh->top_col0 = t0 < ns ? pl->sn[t0].first : pl->m;
  sh->top_rect_off = t0 < ns ? pl->sn[t0].poff : pl->rect;
  sh->top_rect_len = pl->rect - sh->top_rect_off;
  // filtered pair lists for the top: A = owned descendants below t0, B = descendants inside the top
  std::vector<Pair> pA, pB;
  std::vector<int> begA(ns + 1, 0), begB(ns + 1, 0);
  for (int J = 0; J < ns; J++) {
    begA[J] = (int)pA.size(); begB[J] = (int)pB.size();
    if (J < t0) continue;
    for (int e = pl->pair_beg[J]; e < pl->pair_beg[J + 1]; e++) {
      const Pair &p = pairs[e];
      if (p.K >= t0) pB.push_back(p);
      else if (sh->owner[p.K] == rank) pA.push_back(p);
    }
  }
  begA[ns] = (int)pA.size(); begB[ns] = (int)pB.size();
  // schedules
  const int nlev = pl->nlevels;
  sh->own_small.assign(nlev, {}); sh->own_big.assign(nlev, {}); sh->own_all.assign(nlev, {});
  sh->top_small.assign(nlev, {}); sh->top_big.assign(nlev, {}); sh->top_all.assign(nlev, {});
  std::vector<int> lists;
  std::vector<UTile> tiles;
  std::vector<std::vector<UTile>> own_tiles(nlev), top_tiles(nlev);
  std::vector<UTile> topA_tiles;
  auto add_tiles = [&](std::vector<UTile> &v, int s2) {
    const Sn &S = pl->sn[s2];
    for (int c0 = 0; c0 < S.n; c0 += UT_C)
      for (int r0 = (c0 / UT_R) * UT_R; r0 < S.m; r0 += UT_R) v.push_back(UTile{s2, r0, c0});
  };
  for (int s2 = 0; s2 < ns; s2++) {
    const int lv = pl->level_of[s2];
    const bool small = sn_is_small(pl, pl->sn[s2]);
    if (s2 < t0) {
      if (sh->owner[s2] != rank) continue;
      (small ? sh->own_small : sh->own_big)[lv].push_back(s2); sh->own_all[lv].push_back(s2);
      if (pl->pair_beg[s2 + 1] > pl->pair_beg[s2]) add_tiles(own_tiles[lv], s2);
    } else {
      (small ? sh->top_small : sh->top_big)[lv].push_back(s2); sh->top_all[lv].push_back(s2);
      if (begB[s2 + 1] > begB[s2]) add_tiles(top_tiles[lv], s2);
      if (begA[s2 + 1] > begA[s2]) add_tiles(topA_tiles, s2);
    }
  }
  for (int lv = 0; lv < nlev; lv++) {
    sh->own_small_off.push_back((int)lists.size()); for (int v : sh->own_small[lv]) lists.push_back(v);
    sh->own_all_off.push_back((int)lists.size()); for (int v : sh->own_all[lv]) lists.push_back(v);
    sh->top_small_off.push_back((int)lists.size()); for (int v : sh->top_small[lv]) lists.push_back(v);
    sh->top_all_off.push_back((int)lists.size()); for (int v : sh->top_all[lv]) lists.push_back(v);
    sh->own_tile_off.push_back((int)tiles.size()); sh->own_tile_cnt.push_back((int)own_tiles[lv].size());
    tiles.insert(tiles.end(), own_tiles[lv].begin(), own_tiles[lv].end());
    sh->top_tile_off.push_back((int)tiles.size()); sh->top_tile_cnt.push_back((int)top_tiles[lv].size());
    tiles.insert(tiles.end(), top_tiles[lv].begin(), top_tiles[lv].end());
  }
  sh->topA_tile_off = (int)tiles.size(); sh->topA_tile_cnt = (int)topA_tiles.size();
  tiles.insert(tiles.end(), topA_tiles.begin(), topA_tiles.end());
  sh->top_list_off = (int)lists.size();
  for (int s2 = t0; s2 < ns; s2++) lists.push_back(s2);
  sh->top_list_cnt = ns - t0;
  std::vector<int> colmask(pl->m, 0);
  for (int s2 = 0; s2 < ns; s2++) {
    const bool mine = s2 < t0 ? sh->owner[s2] == rank : rank == 0;
    for (int c = 0; c < pl->sn[s2].n; c++) colmask[pl->sn[s2].first + c] = mine ? 1 : 0;
  }
  if (lists.empty()) lists.push_back(0);
  if (tiles.empty()) tiles.push_back(UTile{0, 0, 0});
  if (pA.empty()) pA.push_back(Pair{});
  if (pB.empty()) pB.push_back(Pair{});
  SB_TRY(sh->d_lists.upload(lists)); SB_TRY(sh->d_tiles.upload(tiles));
  {
    std::vector<unsigned char> kA(ns, 0), kB(ns, 0);
    for (int K = 0; K < ns; K++) { kA[K] = (K < t0 && sh->owner[K] == rank) ? 1 : 0; kB[K] = K >= t0 ? 1 : 0; }
    SB_TRY(sh->d_kmaskA.upload(kA)); SB_TRY(sh->d_kmaskB.upload(kB));
  }
  SB_TRY(sh->d_pairsA.upload(pA)); SB_TRY(sh->d_pairsB.upload(pB));
  SB_TRY(sh->d_pair_begA.upload(begA)); SB_TRY(sh->d_pair_begB.upload(begB));
  SB_TRY(sh->d_colmask.upload(colmask));
  SB_CUDA(cudaStreamSynchronize(ctx().stream));
  return 0;
}
// t0: first top supernode; the top occupies rect[top_rect_off, +top_rect_len) and columns [top_col0, m) of the
// permuted index space; colmask_dev[c] = 1 for the columns this rank answers for (its trees; the top on rank 0).
int sb200_chol_shard_info(const sb200_chol_plan *pl, sb_idx *t0, sb_idx *top_rect_off, sb_idx *top_rect_len, sb_idx *top_col0,
                          const int **colmask_dev) {
  SB_CHECK(pl->shard, "shard: sb200_chol_shard_create has not been called");
  *t0 = pl->shard->t0; *top_rect_off = pl->shard->top_rect_off; *top_rect_len = pl->shard->top_rect_len;
  *top_col0 = pl->shard->top_col0; *colmask_dev = pl->shard->d_colmask.p;
  return 0;
}

static int shard_factor_levels(sb200_chol_plan *pl, bool top, sb200_chol_pars pars, double *rect, double *d, int *flag, double *sval) {
  auto *sh = pl->shard;
  cudaStream_t st = ctx().stream;
  const int m = pl->m;
  for (int lv = 0; lv < pl->nlevels; lv++) {
    const int ntile = top ? sh->top_tile_cnt[lv] : sh->own_tile_cnt[lv];
    if (ntile) {
      if (pl->upd_lists)
        update_gather_kernel<<<ntile, 256, 0, st>>>(sh->d_tiles.p + (top ? sh->top_tile_off[lv] : sh->own_tile_off[lv]), pl->d_sn.p, pl->d_upd_ptr.p,
                                                    pl->d_upd_src.p, pl->d_upd_K.p, top ? sh->d_kmaskB.p : nullptr, pl->d_U.p, rect);
      else
      update_kernel<<<ntile, 256, 0, st>>>(sh->d_tiles.p + (top ? sh->top_tile_off[lv] : sh->own_tile_off[lv]), pl->d_sn.p,
                                            top ? sh->d_pairsB.p : pl->d_pairs.p, top ? sh->d_pair_begB.p : pl->d_pair_beg.p, pl->d_rel.p, pl->d_U.p, rect);
      SB_LAUNCH_CHECK_N("update_kernel");
    }
    const auto &small = top ? sh->top_small[lv] : sh->own_small[lv];
    SB_TRY(launch_factor_small(pl, small, sh->d_lists.p + (top ? sh->top_small_off[lv] : sh->own_small_off[lv]), pars, rect, d, flag, sval));
    for (int s2 : (top ? sh->top_big[lv] : sh->own_big[lv])) {
      const Sn &S = pl->sn[s2];
      for (int p0 = 0; p0 < S.n; p0 += NB) {
        int w = std::min(NB, S.n - p0);
        diag_kernel<<<1, 256, 0, st>>>(S, p0, w, rect, d, pl->d_lb.p, pl->d_scal.p, pars.maxu, flag, sval, pl->d_diagX.p, m, pl->d_vscratch.p);
        SB_LAUNCH_CHECK_N("diag_kernel");
        int nrow = S.m - (p0 + w);
        if (nrow > 0) {
          trsm_kernel<<<(nrow + 127) / 128, 128, 0, st>>>(S, p0, w, rect, d);
          SB_LAUNCH_CHECK_N("trsm_kernel");
          int ncol = S.n - (p0 + w);
          if (ncol > 0) {
            dim3 g((nrow + 63) / 64, (ncol + 63) / 64);
            trail_kernel<<<g, 256, 0, st>>>(S, p0, w, rect, d);
            SB_LAUNCH_CHECK_N("trail_kernel");
          }
        }
      }
    }
    // contributions of this level's supernodes (own trees: they feed later own levels and the top; top: later top levels)
    {
      const auto &all = top ? sh->top_all[lv] : sh->own_all[lv];
      SB_TRY(launch_schur(pl, all, sh->d_lists.p + (top ? sh->top_all_off[lv] : sh->own_all_off[lv]), rect, d));
    }
  }
  return 0;
}

// Phase 1: this rank's trees + their contributions to the top panels.  Afterwards the caller sums
// rect[top_rect_off, +top_rect_len) over the ranks (one all-reduce).
int sb200_blkchol_shard_local_dev(sb200_chol_plan *pl, const double *Xpr, const double *absd, sb200_chol_pars pars,
                                  double *rect, double *d, int *flag, double *sval) {
  SB_TRY(ensure_init());
  SB_CHECK(pl->shard, "shard: sb200_chol_shard_create has not been called");
  auto *sh = pl->shard;
  cudaStream_t st = ctx().stream;
  const int m = pl->m;
  SB_CUDA(cudaMemsetAsync(flag, 0, sizeof(int) * m, st));
  SB_CUDA(cudaMemsetAsync(sval, 0, sizeof(double) * m, st));
  SB_CUDA(cudaMemsetAsync(d, 0, sizeof(double) * m, st));
  permuteP_kernel<<<m, 256, 0, st>>>(pl->d_sn.p, pl->d_snode.p, pl->d_lindx.p, pl->d_perm.p, pl->d_Xjc.p, pl->d_Xir.p, Xpr, rect, pl->d_diagX.p);
  SB_LAUNCH_CHECK_N("permuteP_kernel");
  bounds_kernel<<<1, 1024, 0, st>>>(m, pl->d_diagX.p, absd, pl->d_perm.p, pars.abstol, pars.canceltol, pars.maxu, pl->d_lb.p, pl->d_scal.p);
  SB_LAUNCH_CHECK_N("bounds_kernel");
  if (sh->rank != 0 && sh->top_rect_len) SB_CUDA(cudaMemsetAsync(rect + sh->top_rect_off, 0, sizeof(double) * sh->top_rect_len, st));
  SB_TRY(shard_factor_levels(pl, false, pars, rect, d, flag, sval));
  if (sh->topA_tile_cnt) {
    if (pl->upd_lists)
      update_gather_kernel<<<sh->topA_tile_cnt, 256, 0, st>>>(sh->d_tiles.p + sh->topA_tile_off, pl->d_sn.p, pl->d_upd_ptr.p, pl->d_upd_src.p, pl->d_upd_K.p,
                                                              sh->d_kmaskA.p, pl->d_U.p, rect);
    else
    update_kernel<<<sh->topA_tile_cnt, 256, 0, st>>>(sh->d_tiles.p + sh->topA_tile_off, pl->d_sn.p, sh->d_pairsA.p, sh->d_pair_begA.p, pl->d_rel.p, pl->d_U.p, rect);
    SB_LAUNCH_CHECK_N("update_kernel");
  }
  return 0;
}
// Phase 2 (after the all-reduce of the top panels): the top, redundantly on every rank.
int sb200_blkchol_shard_top_dev(sb200_chol_plan *pl, sb200_chol_pars pars, double *rect, double *d, int *flag, double *sval) {
  SB_TRY(ensure_init());
  SB_CHECK(pl->shard, "shard: sb200_chol_shard_create has not been called");
  return shard_factor_levels(pl, true, pars, rect, d, flag, sval);
}

static size_t shard_solve_shm(sb200_chol_plan *pl) { return std::max(fw_shm(pl), sizeof(double) * (size_t)pl->max_sn_n); }
// Forward, phase 1: y = b(perm) (top rows zeroed off rank 0), own trees, pull into the top rows.  Then all-reduce
// y[top_col0 .. m) per right-hand side.
int sb200_fw_shard_local_dev(sb200_chol_plan *pl, const double *rect, const double *b, double *y, sb_idx nrhs) {
  SB_TRY(ensure_init());
  SB_CHECK(pl->shard, "shard: sb200_chol_shard_create has not been called");
  auto *sh = pl->shard;
  cudaStream_t st = ctx().stream;
  const int m = pl->m;
  if (m == 0 || nrhs == 0) return 0;
  const long long tot = (long long)m * nrhs;
  gather_perm_kernel<<<(unsigned)((tot + 255) / 256), 256, 0, st>>>(m, (int)nrhs, pl->d_perm.p, b, y);
  SB_LAUNCH_CHECK_N("gather_perm_kernel");
  if (sh->rank != 0 && sh->top_col0 < m)
    for (sb_idx r = 0; r < nrhs; r++) SB_CUDA(cudaMemsetAsync(y + r * m + sh->top_col0, 0, sizeof(double) * (m - sh->top_col0), st));
  const size_t shm = shard_solve_shm(pl);
  SB_CHECK(shm <= 200 * 1024, "fwblkslv: supernode wider than the shared-memory solve supports (%d)", pl->max_sn_n);
  if (shm > 48 * 1024) SB_CUDA(cudaFuncSetAttribute(fwsolve_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)shm));
  SB_TRY(ensure_cvec(pl, (int)nrhs));
  for (int lv = 0; lv < pl->nlevels; lv++) {
    if (sh->own_all[lv].empty()) continue;
    dim3 g((unsigned)sh->own_all[lv].size(), (unsigned)nrhs);
    fwsolve_kernel<<<g, 512, shm, st>>>(sh->d_lists.p + sh->own_all_off[lv], pl->d_sn.p, pl->d_pull_ptr.p, pl->d_pull_src.p, pl->d_pull_K.p, nullptr, rect, y, m, 1, pl->d_cvec.p, pl->ctot);
    SB_LAUNCH_CHECK_N("fwsolve_kernel");
  }
  if (sh->top_list_cnt) {
    dim3 g((unsigned)sh->top_list_cnt, (unsigned)nrhs);
    fwsolve_kernel<<<g, 512, shm, st>>>(sh->d_lists.p + sh->top_list_off, pl->d_sn.p, pl->d_pull_ptr.p, pl->d_pull_src.p, pl->d_pull_K.p, sh->d_kmaskA.p, rect, y, m, 0, pl->d_cvec.p, pl->ctot);
    SB_LAUNCH_CHECK_N("fwsolve_kernel");
  }
  return 0;
}
// Forward, phase 2 (after the all-reduce of the top segment), ./d on this rank's columns, backward over the top and the
// own trees; foreign columns of z end up zero, so that all-reduce(sum) of z followed by sb200_bw_shard_finish_dev
// gives y = L' \ ((L \ b(perm)) ./ d) in the original order.  z: m x nrhs scratch (the permuted solution).
int sb200_solve_shard_top_dev(sb200_chol_plan *pl, const double *rect, const double *d, const int *flag, double *y, sb_idx nrhs) {
  SB_TRY(ensure_init());
  SB_CHECK(pl->shard, "shard: sb200_chol_shard_create has not been called");
  auto *sh = pl->shard;
  cudaStream_t st = ctx().stream;
  const int m = pl->m;
  if (m == 0 || nrhs == 0) return 0;
  const size_t shm = shard_solve_shm(pl);
  if (shm > 48 * 1024) SB_CUDA(cudaFuncSetAttribute(bwsolve_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)shm));
  for (int lv = 0; lv < pl->nlevels; lv++) {
    if (sh->top_all[lv].empty()) continue;
    dim3 g((unsigned)sh->top_all[lv].size(), (unsigned)nrhs);
    fwsolve_kernel<<<g, 512, shm, st>>>(sh->d_lists.p + sh->top_all_off[lv], pl->d_sn.p, pl->d_pull_ptr.p, pl->d_pull_src.p, pl->d_pull_K.p, sh->d_kmaskB.p, rect, y, m, 1, pl->d_cvec.p, pl->ctot);
    SB_LAUNCH_CHECK_N("fwsolve_kernel");
  }
  const long long tot = (long long)m * nrhs;
  // ./d: the top columns on every rank (needed by the backward pass), own columns; foreign columns become 0
  {
    shard_scale_kernel<<<(unsigned)((tot + 255) / 256), 256, 0, st>>>(m, (int)nrhs, sh->d_colmask.p, sh->top_col0, d, flag, pl->d_lb.p, y);
    SB_LAUNCH_CHECK_N("shard_scale_kernel");
  }
  for (int lv = pl->nlevels - 1; lv >= 0; lv--) {
    if (sh->top_all[lv].empty()) continue;
    dim3 g((unsigned)sh->top_all[lv].size(), (unsigned)nrhs);
    bwsolve_kernel<<<g, 512, shm, st>>>(sh->d_lists.p + sh->top_all_off[lv], pl->d_sn.p, pl->d_lindx.p, rect, y, m);
    SB_LAUNCH_CHECK_N("bwsolve_kernel");
  }
  for (int lv = pl->nlevels - 1; lv >= 0; lv--) {
    if (sh->own_all[lv].empty()) continue;
    dim3 g((unsigned)sh->own_all[lv].size(), (unsigned)nrhs);
    bwsolve_kernel<<<g, 512, shm, st>>>(sh->d_lists.p + sh->own_all_off[lv], pl->d_sn.p, pl->d_lindx.p, rect, y, m);
    SB_LAUNCH_CHECK_N("bwsolve_kernel");
  }
  shard_mask_kernel<<<(unsigned)((tot + 255) / 256), 256, 0, st>>>(m, (int)nrhs, sh->d_colmask.p, y);
  SB_LAUNCH_CHECK_N("shard_mask_kernel");
  return 0;
}
// After the all-reduce of z: back to the original order.
int sb200_bw_shard_finish_dev(sb200_chol_plan *pl, const double *z, double *y, sb_idx nrhs) {
  SB_TRY(ensure_init());
  const long long tot = (long long)pl->m * nrhs;
  if (tot == 0) return 0;
  scatter_perm_kernel<<<(unsigned)((tot + 255) / 256), 256, 0, ctx().stream>>>(pl->m, (int)nrhs, pl->d_perm.p, z, y);
  SB_LAUNCH_CHECK_N("scatter_perm_kernel");
  return 0;
}

// The whole sharded factorisation / solve with the collectives issued by the library itself (comm.cu) on the library
// stream: a host calls these like the unsharded entries, on every rank, and the sequence is capturable as one graph.
int sb200_blkchol_sharded_dev(sb200_chol_plan *pl, const double *Xpr, const double *absd, sb200_chol_pars pars,
                              double *rect, double *d, int *flag, double *sval) {
  SB_TRY(sb200_blkchol_shard_local_dev(pl, Xpr, absd, pars, rect, d, flag, sval));
  if (pl->shard->top_rect_len) SB_TRY(sb200_allreduce_sum_dev(rect + pl->shard->top_rect_off, pl->shard->top_rect_len));
  return sb200_blkchol_shard_top_dev(pl, pars, rect, d, flag, sval);
}
int sb200_ldl_solve_sharded_dev(sb200_chol_plan *pl, const double *rect, const double *d, const int *flag,
                                const double *b, double *w, double *y, sb_idx nrhs) {
  SB_TRY(sb200_fw_shard_local_dev(pl, rect, b, w, nrhs));
  const int m = pl->m, c0 = pl->shard->top_col0;
  if (c0 < m)                      // only the top segment of each right-hand side is a sum over ranks
    for (sb_idx r = 0; r < nrhs; r++) SB_TRY(sb200_allreduce_sum_dev(w + r * m + c0, m - c0));
  SB_TRY(sb200_solve_shard_top_dev(pl, rect, d, flag, w, nrhs));
  SB_TRY(sb200_allreduce_sum_dev(w, (sb_idx)m * nrhs));
  return sb200_bw_shard_finish_dev(pl, w, y, nrhs);
}

}  // extern "C"

// --------------------------------------------------------------------------- plan cache
namespace sb {
struct PlanCache {
  std::map<Hash128, sb200_chol_plan *> plans;
  uint64_t clock = 0;
  ~PlanCache() { /* plans leak at process exit on purpose: the CUDA context may be gone */ }
};
static PlanCache g_cache;

static Hash128 structure_key(sb_idx m, sb_idx nsuper, const sb_idx *xsuper, const sb_idx *Ljc, const sb_idx *Lir,
                              const sb_idx *perm, const sb_idx *Xjc, const sb_idx *Xir) {
  Hash128 h = fnv1a(&m, sizeof m);
  h = fnv1a(&nsuper, sizeof nsuper, h);
  h = fnv1a(xsuper, sizeof(sb_idx) * (nsuper + 1), h);
  h = fnv1a(Ljc, sizeof(sb_idx) * (m + 1), h);
  h = fnv1a(Lir, sizeof(sb_idx) * Ljc[m], h);
  h = fnv1a(perm, sizeof(sb_idx) * m, h);
  if (Xjc) { h = fnv1a(Xjc, sizeof(sb_idx) * (m + 1), h); h = fnv1a(Xir, sizeof(sb_idx) * Xjc[m], h); }
  return h;
}

// Find or build the plan for this symbolic structure.  For the solves X's pattern is not
// needed; a plan created without it (Xjc == NULL) gets an empty X pattern.
int get_plan(sb200_chol_plan **out, sb_idx m, sb_idx nsuper, const sb_idx *xsuper, const sb_idx *Ljc,
             const sb_idx *Lir, const sb_idx *perm, const sb_idx *Xjc, const sb_idx *Xir) {
  SB_TRY(ensure_init());
  Hash128 key = structure_key(m, nsuper, xsuper, Ljc, Lir, perm, Xjc, Xir);
  auto it = g_cache.plans.find(key);
  if (it != g_cache.plans.end()) { it->second->cache_stamp = ++g_cache.clock; *out = it->second; return 0; }
  std::vector<sb_idx> zjc;
  if (!Xjc) { zjc.assign(m + 1, 0); Xjc = zjc.data(); Xir = zjc.data(); }
  sb200_chol_plan *pl = nullptr;
  SB_TRY(sb200_chol_plan_create(&pl, m, nsuper, xsuper, Ljc, Lir, perm, Xjc, Xir));
  pl->key = key;
  // bounded, least-recently-used first.  Plans of this cache are only ever borrowed for the duration of one host
  // entry (device-resident callers own theirs through sb200_chol_plan_create), and destroying a plan frees device
  // memory, which waits for the kernels still using it.
  while (g_cache.plans.size() >= 16) {
    auto lru = g_cache.plans.begin();
    for (auto i2 = g_cache.plans.begin(); i2 != g_cache.plans.end(); ++i2)
      if (i2->second->cache_stamp < lru->second->cache_stamp) lru = i2;
    cudaStreamSynchronize(ctx().stream);
    sb200_chol_plan_destroy(lru->second);
    g_cache.plans.erase(lru);
  }
  pl->cache_stamp = ++g_cache.clock;
  g_cache.plans[key] = pl;
  *out = pl;
  return 0;
}
}  // namespace sb

extern "C" {

static double now_ms() {
  struct timespec ts; clock_gettime(CLOCK_MONOTONIC, &ts);
  return ts.tv_sec * 1e3 + ts.tv_nsec * 1e-6;
}

int sb200_blkchol(sb_idx m, sb_idx nsuper, const sb_idx *xsuper, const sb_idx *Ljc, const sb_idx *Lir,
                  const sb_idx *perm, const sb_idx *Xjc, const sb_idx *Xir, const double *Xpr,
                  const double *absd, sb200_chol_pars pars, double *Lpr_out, double *d_out,
                  sb_idx *skip_idx, double *skip_val, sb_idx *nskip, sb_idx *add_idx, double *add_val,
                  sb_idx *nadd) {
  const bool trace = getenv("SB200_TRACE") != nullptr;
  double t0 = now_ms();
  sb200_chol_plan *pl = nullptr;
  SB_TRY(get_plan(&pl, m, nsuper, xsuper, Ljc, Lir, perm, Xjc, Xir));
  double t1 = now_ms();
  *nskip = 0; *nadd = 0;
  if (m == 0) return 0;
  arena_reset();
  cudaStream_t st = ctx().stream;
  const size_t nnzX = (size_t)Xjc[m];
  double *dX = (double *)mirror_input(Xpr, sizeof(double) * nnzX), *dabsd = arena<double>((size_t)m), *drect = arena<double>((size_t)pl->rect),
         *dd = arena<double>((size_t)m), *dsval = arena<double>((size_t)m), *dL = arena<double>((size_t)pl->nnzL);
  int *dflag = arena<int>((size_t)m);
  SB_CHECK(dX && dabsd && drect && dd && dsval && dL && dflag, "blkchol: out of device memory");
  if (absd) SB_CUDA(cudaMemcpyAsync(dabsd, absd, sizeof(double) * m, cudaMemcpyHostToDevice, st));
  double t2 = now_ms();
  SB_TRY(sb200_blkchol_dev(pl, dX, absd ? dabsd : nullptr, pars, drect, dd, dflag, dsval));
  SB_TRY(sb200_chol_rect_to_csc_dev(pl, drect, dflag, dL));
  if (trace) cudaStreamSynchronize(st);
  double t3 = now_ms();
  std::vector<int> flag(m);
  std::vector<double> sval(m);
  SB_CUDA(cudaMemcpyAsync(Lpr_out, dL, sizeof(double) * pl->nnzL, cudaMemcpyDeviceToHost, st));
  SB_CUDA(cudaMemcpyAsync(d_out, dd, sizeof(double) * m, cudaMemcpyDeviceToHost, st));
  SB_CUDA(cudaMemcpyAsync(flag.data(), dflag, sizeof(int) * m, cudaMemcpyDeviceToHost, st));
  SB_CUDA(cudaMemcpyAsync(sval.data(), dsval, sizeof(double) * m, cudaMemcpyDeviceToHost, st));
  SB_CUDA(cudaStreamSynchronize(st));
  double t4 = now_ms();
  for (int j = 0; j < m; j++) {
    if (flag[j] == 1) { skip_idx[*nskip] = j; skip_val[*nskip] = sval[j]; (*nskip)++; }
    else if (flag[j] == 2) { add_idx[*nadd] = j; add_val[*nadd] = sval[j]; (*nadd)++; }
  }
  if (trace) fprintf(stderr, "[sb200_blkchol] plan %.3f ms, h2d %.3f, factor %.3f, d2h %.3f\n", t1 - t0, t2 - t1, t3 - t2, t4 - t3);
  return 0;
}

static int solve_host(bool fw, sb_idx m, sb_idx nsuper, const sb_idx *xsuper, const sb_idx *Ljc, const sb_idx *Lir,
                      const double *Lpr, const sb_idx *perm, const double *b, double *y, sb_idx nrhs) {
  sb200_chol_plan *pl = nullptr;
  SB_TRY(get_plan(&pl, m, nsuper, xsuper, Ljc, Lir, perm, nullptr, nullptr));
  if (m == 0 || nrhs == 0) return 0;
  arena_reset();
  cudaStream_t st = ctx().stream;
  // The factor values usually repeat over many solves (3-4 solves x fw/bw per IPM iteration): keep the
  // device copy in the internal layout (+ inverted diagonal blocks, L') under a content hash.
  const Hash128 hL = hash128(Lpr, sizeof(double) * pl->nnzL);
  if (!(pl->Lcache_valid && pl->Lcache_hash == hL)) {
    double *dL = arena<double>((size_t)pl->nnzL);
    SB_CHECK(dL, "solve: out of device memory");
    if (pl->d_rect_cache.n < (size_t)pl->rect) SB_TRY(pl->d_rect_cache.alloc((size_t)pl->rect));
    SB_CUDA(cudaMemcpyAsync(dL, Lpr, sizeof(double) * pl->nnzL, cudaMemcpyHostToDevice, st));
    SB_TRY(sb200_chol_csc_to_rect_dev(pl, dL, pl->d_rect_cache.p));
    if (pl->dense_fast) SB_TRY(dense_compute_dinv(pl, pl->d_rect_cache.p));
    pl->Lcache_hash = hL; pl->Lcache_valid = true;
  }
  double *db = arena<double>((size_t)(m * nrhs)), *dy = arena<double>((size_t)(m * nrhs));
  SB_CHECK(db && dy, "solve: out of device memory");
  SB_CUDA(cudaMemcpyAsync(db, b, sizeof(double) * m * nrhs, cudaMemcpyHostToDevice, st));
  if (fw) SB_TRY(sb200_fwblkslv_dev(pl, pl->d_rect_cache.p, db, dy, nrhs));
  else SB_TRY(sb200_bwblkslv_dev(pl, pl->d_rect_cache.p, db, dy, nrhs));
  SB_CUDA(cudaMemcpyAsync(y, dy, sizeof(double) * m * nrhs, cudaMemcpyDeviceToHost, st));
  SB_CUDA(cudaStreamSynchronize(st));
  return 0;
}

int sb200_fwblkslv(sb_idx m, sb_idx nsuper, const sb_idx *xsuper, const sb_idx *Ljc, const sb_idx *Lir,
                   const double *Lpr, const sb_idx *perm, const double *b, double *y, sb_idx nrhs) {
  return solve_host(true, m, nsuper, xsuper, Ljc, Lir, Lpr, perm, b, y, nrhs);
}
int sb200_bwblkslv(sb_idx m, sb_idx nsuper, const sb_idx *xsuper, const sb_idx *Ljc, const sb_idx *Lir,
                   const double *Lpr, const sb_idx *perm, const double *b, double *y, sb_idx nrhs) {
  return solve_host(false, m, nsuper, xsuper, Ljc, Lir, Lpr, perm, b, y, nrhs);
}

// Sparse right-hand sides: densify on the host side of the boundary, solve, and pick the
// entries of the symbolic pattern (mathematically identical to selfwsolve, which merely skips
// supernodes that provably stay zero: fwblkslv.c:150-183).
static int solve_sparse(sb_idx m, sb_idx nsuper, const sb_idx *xsuper, const sb_idx *Ljc, const sb_idx *Lir,
                        const double *Lpr, const sb_idx *perm, sb_idx nrhs, const sb_idx *bjc, const sb_idx *bir,
                        const double *bpr, const sb_idx *yjc, const sb_idx *yir, double *ypr) {
  std::vector<double> B((size_t)(m * nrhs), 0.0), Y((size_t)(m * nrhs), 0.0);
  {
    for (sb_idx j = 0; j < nrhs; j++)
      for (sb_idx k = bjc[j]; k < bjc[j + 1]; k++) B[(size_t)(j * m + bir[k])] = bpr[k];
    SB_TRY(solve_host(true, m, nsuper, xsuper, Ljc, Lir, Lpr, perm, B.data(), Y.data(), nrhs));
    for (sb_idx j = 0; j < nrhs; j++)
      for (sb_idx k = yjc[j]; k < yjc[j + 1]; k++) ypr[k] = Y[(size_t)(j * m + yir[k])];
  }
  return 0;
}
int sb200_fwblkslv_sparse(sb_idx m, sb_idx nsuper, const sb_idx *xsuper, const sb_idx *Ljc, const sb_idx *Lir,
                          const double *Lpr, const sb_idx *perm, sb_idx nrhs, const sb_idx *bjc, const sb_idx *bir,
                          const double *bpr, const sb_idx *yjc, const sb_idx *yir, double *ypr) {
  return solve_sparse(m, nsuper, xsuper, Ljc, Lir, Lpr, perm, nrhs, bjc, bir, bpr, yjc, yir, ypr);
}
}  // extern "C"
