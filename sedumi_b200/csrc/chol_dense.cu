// chol_dense.cu -- fast path for a factor that is ONE dense supernode (every shipped SeDuMi example
// and every dense-ADA problem: symbchol.m:71-78 builds L = tril(ones) with a single supernode).
//
// At these sizes (m = 123..5000) the reference's column-serial LDL' is latency-bound, and so is a
// naive GPU port (one launch per panel step: 3 launches x m/32 panels).  This file restructures it:
//
//  * dense_factor: ONE persistent cooperative kernel.  Per 32-column panel: CTA 0 factors the 32x32
//    diagonal block warp-synchronously in shared memory, applying SeDuMi's pivot rules
//    (blkchol2.c:96-167; the rare stability test pulls in the whole CTA); one grid barrier; then every
//    CTA takes 64x64 tiles of the trailing matrix, re-derives the two row slabs of L21 it needs from
//    the untouched panel columns (row-parallel triangular solve in registers) and applies the
//    rank-32 update -- no second barrier between "TRSM" and "SYRK".  L is written to a separate
//    output array, so panel columns are never overwritten while other CTAs still read them.
//    The inverses of the 32x32 unit-lower diagonal blocks are produced at the end for the solves.
//
//  * dense_fwsolve / dense_bwsolve: dataflow triangular solves.  Warp b owns block-row b: it
//    accumulates L(b, j) * y_j for j < b as the y_j are published (flags), then applies the inverted
//    diagonal block.  The critical path per 32 rows is two 32x32 mat-vecs and a flag hand-off
//    instead of a 32-step substitution; the other warps stream the rest of L concurrently.
//    (fwblkslv.c:77-134 / bwblkslv.c:73-125 semantics: y = L\b(perm), y(perm) = L'\b.)
#include <cooperative_groups.h>
#include <stdlib.h>
#include "chol_plan.h"

namespace sb {

static const int PB = 32;          // panel width
static const int TS = 64;          // trailing tile edge

struct ArgMaxD { double v; int i; };
__device__ __forceinline__ ArgMaxD amd_better(ArgMaxD a, ArgMaxD b) {
  if (b.v > a.v || (b.v == a.v && b.i < a.i)) return b;
  return a;
}
__device__ __forceinline__ ArgMaxD block_argmax_d(ArgMaxD x, ArgMaxD *sh) {
  for (int o = 16; o > 0; o >>= 1) {
    ArgMaxD y; y.v = __shfl_down_sync(0xffffffffu, x.v, o); y.i = __shfl_down_sync(0xffffffffu, x.i, o);
    x = amd_better(x, y);
  }
  int w = threadIdx.x >> 5, l = threadIdx.x & 31, nw = (blockDim.x + 31) >> 5;
  __syncthreads();
  if (l == 0) sh[w] = x;
  __syncthreads();
  if (w == 0) {
    x = (l < nw) ? sh[l] : ArgMaxD{-1.0, 0x7fffffff};
    for (int o = 16; o > 0; o >>= 1) {
      ArgMaxD y; y.v = __shfl_down_sync(0xffffffffu, x.v, o); y.i = __shfl_down_sync(0xffffffffu, x.i, o);
      x = amd_better(x, y);
    }
    if (l == 0) sh[0] = x;
  }
  __syncthreads();
  x = sh[0];
  __syncthreads();
  return x;
}

// tile t of the lower-triangular tile grid, row-major: t = ti(ti+1)/2 + tj, tj <= ti
__device__ __forceinline__ void tile_of(int t, int &ti, int &tj) {
  ti = (int)((sqrt(8.0 * t + 1.0) - 1.0) * 0.5);
  while ((ti + 1) * (ti + 2) / 2 <= t) ti++;
  while (ti * (ti + 1) / 2 > t) ti--;
  tj = t - ti * (ti + 1) / 2;
}

__device__ __forceinline__ void grid_barrier(unsigned *ctr, unsigned target) {
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence();
    atomicAdd(ctr, 1u);
    while (*((volatile unsigned *)ctr) < target) { }
    __threadfence();
  }
  __syncthreads();
}

// W: working matrix (m x m, ld = m, lower triangle live); Lo: output factor (same layout).
__global__ void __launch_bounds__(256)
dense_ldl_kernel(int m, double *W, double *Lo, double *d, const double *lb, const double *scal, double maxu,
                 int *flag, double *sval, const double *diagX, double *vscratch, double *dinv, unsigned *bar, long long *tdbg) {
  __shared__ double A[PB][PB + 1];
  __shared__ double s_lb[PB], z[PB], dloc[PB];
  __shared__ int skipped[PB];
  __shared__ ArgMaxD sh_am[32];
  __shared__ double s_x;
  __shared__ int s_state;
  __shared__ double As[PB][TS + 1], Bs[PB][TS + 1];
  const int ld = m;
  const double ub = scal[0];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  unsigned bar_target = 0;
  const int npanels = (m + PB - 1) / PB;
  volatile unsigned *la_fail = bar + 4;            // la_fail[pi] = 1: the look-ahead factorisation of panel pi gave up
  // ------------------------------------------------------------------ phase A: diagonal block of panel pi (one CTA)
  // allow_test = false (look-ahead, the rows below the block are still being updated by the other
  // CTAs): returns false as soon as a pivot needs the reference's stability test, nothing published.
  auto phaseA = [&](const int pi, const bool allow_test, const bool preloaded) -> bool {
    const int p0 = pi * PB, w = min(PB, m - p0), base = p0 + w;
    {
      if (!preloaded) for (int idx = tid; idx < PB * PB; idx += blockDim.x) {
        int r = idx % PB, c = idx / PB;
        A[r][c] = (r < w && c < w && r >= c) ? W[(long long)(p0 + c) * ld + p0 + r] : 0.0;
      }
      if (tid < PB) { skipped[tid] = 0; dloc[tid] = 0.0; }
      __syncthreads();
      if (tid < PB) s_lb[tid] = (tid < w) ? lb[p0 + tid] : 0.0;
      __syncthreads();
      int k_resume = 0, resolved_k = -1;
      // All 8 warps cooperate on each pivot step: the lower triangle below/right of the pivot is at most 31*32/2
      // elements, one per thread.  (One warp holding the block in registers with the pivot column moved by shuffles --
      // ldl_block.cuh, used by the supernodal kernel -- is slower as part of THIS kernel: the single warp is
      // issue-bound on 31 shuffle/multiply/FMA triples per pivot.)
      while (true) {
        {
        int k = k_resume;
        for (; k < w; k++) {
          const int gk = p0 + k;
          double xkk = A[k][k];
          const bool resolved = (k == resolved_k);
          if (resolved) xkk = s_x;
          const bool skip = !(xkk > s_lb[k]);
          if (!skip && !resolved && (m - gk > 1) && (xkk < ub)) break;          // stability test needed (uniform)
          if (skip) {
            if (tid == 0) { flag[gk] = 1; sval[gk] = xkk; skipped[k] = 1; dloc[k] = 0.0; }
            continue;
          }
          const double rinv = 1.0 / xkk;
          // element (r,c), k < c <= r < w: A[r][c] -= (A[c][k]/xkk) * A[r][k]
          {
            const int r = lane;                                   // warp wq handles columns k+1+wq, +8, ...
            const double xr = (r > k && r < w) ? A[r][k] : 0.0;
            for (int c = k + 1 + warp; c < w; c += 8)
              if (r >= c && r < w) A[r][c] -= (A[c][k] * rinv) * xr;
          }
          __syncthreads();
          // (scaling the column one step later, in the shadow of the next update, saves a barrier but
          // is slower: the extra loop-carried state lengthens the dependent chain)
          if (tid > k && tid < w) A[tid][k] *= rinv;
          if (tid == 0) { dloc[k] = xkk; A[k][k] = 1.0; }
          __syncthreads();
        }
        if (tid == 0) s_state = k;
        }
        __syncthreads();
        const int k = s_state;
        if (k >= w) break;
        if (!allow_test) return false;               // uniform: s_state is shared
        // ---- stability test for column k (rare): the reference compares x_kk with |x[idamax+1]|/maxu
        // (blkchol2.c:66-70,122); needs the fully updated sub-column, i.e. the tail rows as well.
        {
          const int gk = p0 + k;
          double xkk = A[k][k];
          const int collen = m - gk;
          if (tid == 0) {
            z[k] = 1.0;
            for (int i = k - 1; i >= 0; i--) {
              double acc = 0.0;
              if (!skipped[i]) for (int j = i + 1; j <= k; j++) acc += A[j][i] * z[j];
              z[i] = -acc;
            }
          }
          __syncthreads();
          ArgMaxD am{-1.0, 0x7fffffff};
          for (int r = k + 1 + tid; r < w; r += blockDim.x) am = amd_better(am, ArgMaxD{fabs(A[r][k]), r - (k + 1)});
          for (int r = base + tid; r < m; r += blockDim.x) {
            double v = 0.0;
            for (int j = 0; j <= k; j++) v += W[(long long)(p0 + j) * ld + r] * z[j];
            vscratch[r] = v;
            am = amd_better(am, ArgMaxD{fabs(v), r - (gk + 1)});
          }
          am = block_argmax_d(am, sh_am);
          if (tid == 0) {
            const int t = am.i + 1, sublen = collen - 1;
            double v;
            if (t < sublen) {
              int r = gk + 1 + t;
              v = (r < base) ? A[r - p0][k] : vscratch[r];
            } else if (k + 1 < w) {
              v = A[k + 1][k + 1];
            } else if (base < m) {
              // diagonal of the next panel's first column as the reference holds it at this moment
              const int r = base;
              double u[PB];
              double x = W[(long long)r * ld + r];
              for (int j = 0; j < k; j++) {
                double uj = W[(long long)(p0 + j) * ld + r];
                for (int i = 0; i < j; i++) if (!skipped[i]) uj -= u[i] * A[j][i];
                u[j] = uj;
                if (!skipped[j]) x -= uj * uj / dloc[j];
              }
              v = x;
            } else v = 0.0;
            const double ubk = fabs(v) / maxu;
            if (xkk < ubk) { flag[gk] = 2; sval[gk] = ubk - xkk; xkk = ubk; }
            s_x = xkk;
          }
          __syncthreads();
          resolved_k = k; k_resume = k;
        }
      }
      if (tdbg && tid == 0) tdbg[pi * 8 + 2] = clock64();
      // publish d and L11 (unit lower; skipped columns zeroed) into the outputs
      if (tid < w) d[p0 + tid] = dloc[tid];
      for (int idx = tid; idx < w * w; idx += blockDim.x) {
        int r = idx % w, c = idx / w;
        if (r >= c) Lo[(long long)(p0 + c) * ld + p0 + r] = (r == c) ? 1.0 : (skipped[c] ? 0.0 : A[r][c]);
      }
    }
    return true;
  };
  if (tdbg && blockIdx.x == 0 && tid == 0) tdbg[0] = clock64();
  if (blockIdx.x == 0) phaseA(0, true, false);
  if (tdbg && blockIdx.x == 0 && tid == 0) tdbg[3] = clock64();
  bar_target += gridDim.x;
  grid_barrier(bar, bar_target);
  for (int pi = 0; pi < npanels; pi++) {
    const int p0 = pi * PB, w = min(PB, m - p0), base = p0 + w;
    const int nrow = m - base;
    const int nslab = nrow > 0 ? (nrow + TS - 1) / TS : 0;
    const int ntiles = nslab * (nslab + 1) / 2;
    if (tdbg && blockIdx.x == 0 && tid == 0) tdbg[pi * 8 + 4] = clock64();
    // ------------------------------------------------------------------ phase B: trailing tiles, and on CTA 0
    // (which owns the tile holding the next diagonal block) the look-ahead factorisation of panel pi+1
    if (nrow > 0) {
      // L11 (strictly lower) and d of this panel -> shared (A / dloc are reused as scratch by every CTA).
      // The panel CTA factored this block itself a moment ago: A and dloc still hold it.
      const bool solo = gridDim.x == 1;
      if (solo || blockIdx.x != 0) {
        for (int idx = tid; idx < PB * PB; idx += blockDim.x) {
          int r = idx % PB, c = idx / PB;
          A[r][c] = (r < w && c < w && r > c) ? Lo[(long long)(p0 + c) * ld + p0 + r] : 0.0;
        }
        if (tid < PB) dloc[tid] = (tid < w) ? d[p0 + tid] : 0.0;
      }
      __syncthreads();
      if (tid < PB) s_lb[tid] = (dloc[tid] > 0.0) ? 1.0 / dloc[tid] : 0.0;        // reciprocal pivots (0 marks a skipped pivot)
      __syncthreads();
      // with more than one CTA, CTA 0 is the dedicated panel CTA (look-ahead below) and takes no tile
      const int t_first = solo ? 0 : (blockIdx.x == 0 ? ntiles : (int)blockIdx.x - 1);
      const int t_step = solo ? 1 : (int)gridDim.x - 1;
      for (int t = t_first; t < ntiles; t += t_step) {
        int ti, tj; tile_of(t, ti, tj);
        if (tid < 2 * TS) {
          const bool isB = tid >= TS;
          const int lr = isB ? tid - TS : tid;
          const int r = base + (isB ? tj : ti) * TS + lr;
          double a[PB];
          if (r < m) {
#pragma unroll
            for (int j = 0; j < PB; j++) a[j] = (j < w) ? W[(long long)(p0 + j) * ld + r] : 0.0;
#pragma unroll
            for (int j = 0; j < PB; j++) {
              const double rj = s_lb[j];
              const double xj = a[j];
              if (rj > 0.0) {
#pragma unroll
                for (int j2 = j + 1; j2 < PB; j2++) a[j2] -= xj * A[j2][j];
                a[j] = xj * rj;
              } else a[j] = 0.0;
            }
          } else {
#pragma unroll
            for (int j = 0; j < PB; j++) a[j] = 0.0;
          }
          if (!isB) {
#pragma unroll
            for (int j = 0; j < PB; j++) As[j][lr] = a[j];
            if (tj == 0 && r < m) {
#pragma unroll
              for (int j = 0; j < PB; j++) if (j < w) Lo[(long long)(p0 + j) * ld + r] = a[j];
            }
          } else {
#pragma unroll
            for (int j = 0; j < PB; j++) Bs[j][lr] = a[j] * dloc[j];
          }
        }
        __syncthreads();
        {
          const int tx = tid % 16, ty = tid / 16;
          double acc[4][4] = {};
#pragma unroll 8
          for (int j = 0; j < PB; j++) {
            double av[4], bv[4];
#pragma unroll
            for (int i = 0; i < 4; i++) { av[i] = As[j][tx + 16 * i]; bv[i] = Bs[j][ty + 16 * i]; }
#pragma unroll
            for (int i = 0; i < 4; i++)
#pragma unroll
              for (int q = 0; q < 4; q++) acc[i][q] += av[i] * bv[q];
          }
          const int r0 = base + ti * TS, c0 = base + tj * TS;
          const bool lead_skip = !solo && t == 0;
#pragma unroll
          for (int q = 0; q < 4; q++) {
            const int c = c0 + ty + 16 * q;
            if (c < m) {
#pragma unroll
              for (int i = 0; i < 4; i++) {
                const int r = r0 + tx + 16 * i;
                // the leading PB x PB block of tile 0 belongs to the panel CTA (look-ahead below)
                if (r < m && r >= c && !(lead_skip && r < base + PB && c < base + PB)) W[(long long)c * ld + r] -= acc[i][q];
              }
            }
          }
        }
        __syncthreads();
      }
      if (tdbg && blockIdx.x == 0 && tid == 0) tdbg[pi * 8 + 1] = clock64();
      if (blockIdx.x == 0 && pi + 1 < npanels) {
        // look-ahead: factor the next diagonal block while the other CTAs update the trailing matrix.
        bool pre = false;
        if (!solo) {
          // The block is formed here from the not yet updated W (some other CTA updates W itself as part
          // of tile 0), with the same operation order as the tile code: rows base..base+wn-1 of L21, then
          // W(blk) - L21 D L21'.
          const int wn = min(PB, m - base);
          // all global loads first: 4 panel entries (row r, columns sub+8i) and 4 entries of the block per thread
          const int rr = tid >> 3, sub = tid & 7;
          double a[4], vpre[4];
#pragma unroll
          for (int i = 0; i < 4; i++) {
            const int c = sub + 8 * i;
            a[i] = (rr < wn && c < w) ? W[(long long)(p0 + c) * ld + base + rr] : 0.0;
          }
#pragma unroll
          for (int i = 0; i < 4; i++) {
            const int idx = tid + 256 * i, r = idx % PB, c = idx / PB;
            vpre[i] = (r < wn && c < wn && r >= c) ? W[(long long)(base + c) * ld + base + r] : 0.0;
          }
          // forward substitution along the row, 8 lanes per row; same operations per element as the tile code
#pragma unroll
          for (int j = 0; j < PB; j++) {
            const double rj = s_lb[j];
            const double xj = __shfl_sync(0xffffffffu, a[j >> 3], (lane & ~7) | (j & 7));
            if (rj > 0.0) {
#pragma unroll
              for (int i = 0; i < 4; i++) {
                const int c = sub + 8 * i;
                if (c > j) a[i] -= xj * A[c][j];
              }
              if (sub == (j & 7)) a[j >> 3] = xj * rj;
            } else if (sub == (j & 7)) a[j >> 3] = 0.0;
          }
#pragma unroll
          for (int i = 0; i < 4; i++) {
            const int c = sub + 8 * i;
            As[c][rr] = a[i];
            Bs[c][rr] = a[i] * dloc[c];
          }
          __syncthreads();
#pragma unroll
          for (int i = 0; i < 4; i++) {
            const int idx = tid + 256 * i, r = idx % PB, c = idx / PB;
            double v = 0.0;
            if (r < wn && c < wn && r >= c) {
              double acc = 0.0;
#pragma unroll 8
              for (int j = 0; j < PB; j++) acc += As[j][r] * Bs[j][c];
              v = vpre[i] - acc;
              W[(long long)(base + c) * ld + base + r] = v;      // sole writer of this block (the tile code skips it)
            }
            A[r][c] = v;
          }
          __syncthreads();
          pre = true;
        }
        const bool ok = phaseA(pi + 1, false, pre);
        if (!ok && tid == 0) la_fail[pi + 1] = 1u;
      }
    }
    if (tdbg && blockIdx.x == 0 && tid == 0) tdbg[pi * 8 + 5] = clock64();
    bar_target += gridDim.x;
    grid_barrier(bar, bar_target);
    if (tdbg && blockIdx.x == 0 && tid == 0) tdbg[pi * 8 + 6] = clock64();
    if (pi + 1 < npanels && la_fail[pi + 1]) {     // rare: a pivot of the next panel needs the stability test,
      if (blockIdx.x == 0) phaseA(pi + 1, true, false);   // which reads the fully updated rows below the block
      bar_target += gridDim.x;
      grid_barrier(bar, bar_target);
    }
  }
  // ------------------------------------------------------------------ inverses of the diagonal blocks
  for (int pi = blockIdx.x; pi < npanels; pi += gridDim.x) {
    const int p0 = pi * PB, w = min(PB, m - p0);
    for (int idx = tid; idx < PB * PB; idx += blockDim.x) {
      int r = idx % PB, c = idx / PB;
      A[r][c] = (r < w && c < w && r > c) ? Lo[(long long)(p0 + c) * ld + p0 + r] : 0.0;
    }
    __syncthreads();
    if (warp == 0) {
      // lane c: column c of inv(L11) by forward substitution, x kept in registers
      double x[PB];
#pragma unroll
      for (int i = 0; i < PB; i++) x[i] = (i == lane) ? 1.0 : 0.0;
#pragma unroll
      for (int i = 1; i < PB; i++) {
        double acc = 0.0;
#pragma unroll
        for (int j = 0; j < PB; j++) if (j < i) acc += A[i][j] * x[j];
        x[i] -= acc;                                   // rows above the diagonal stay 0 since x[j]=0 for j<lane
      }
      double *out = dinv + (long long)pi * PB * PB + lane * PB;
#pragma unroll
      for (int i = 0; i < PB; i++) out[i] = x[i];      // column-major: column = lane
    }
    __syncthreads();
  }
}

// ---------------------------------------------------------------------------------- solves
// One CTA of 32 warps per right-hand side.  Warp b owns block rows b, b+32, ... (ascending), y and
// the ready flags live in shared memory when the whole vector fits (m <= 8192), else in global.
__device__ __forceinline__ void cp_async8(void *smem_dst, const void *gsrc) {
  unsigned sa = (unsigned)__cvta_generic_to_shared(smem_dst);
  asm volatile("cp.async.ca.shared.global [%0], [%1], 8;\n" ::"r"(sa), "l"(gsrc) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;\n" ::: "memory"); }
template <int N> __device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;\n" ::"n"(N) : "memory"); }

// Dataflow triangular solve.  A thread-block CLUSTER of CL CTAs x 8 warps works on one right-hand side;
// warp g of the cluster (g = warp*CL + cta rank) owns block rows g, g+8*CL, ... (ascending in solve order).
// For its block row it walks the already-solved blocks j; the 32x32 block L(b, j) is staged through a
// private 2-deep cp.async ring in shared memory, so the global-load latency of block j+1/j+2 hides behind
// the wait for y_j and the FMAs.  A solved y_b is broadcast into the shared memory of every CTA of the
// cluster (distributed shared memory) followed by its ready flag, so the consumers poll local shared
// memory: the dependent chain costs one DSMEM store per block row instead of a trip through L2, and
// the factor streams through CL SMs instead of one (one CTA pulls ~40 GB/s here; the solve of m=666
// was bound by exactly that).  CL = 1 is the plain single-CTA kernel.
// BACKWARD reads the transposed factor, which makes both directions the same coalesced stream.
static const int SOLVE_WARPS = 8;
static const int SOLVE_CLUSTER = 8;
__device__ __forceinline__ void fence_cluster() { asm volatile("fence.acq_rel.cluster;\n" ::: "memory"); }
// Hand-over of a solved block row inside the cluster: the producer writes y_b into every CTA's shared memory with
// st.async, which also counts the bytes on an mbarrier of the RECEIVING CTA; consumers sleep on their local mbarrier
// (try_wait is a hardware wait, not a poll).  One DSMEM hop + wake-up per dependent block row,
// instead of store + cluster fence + flag + polling.
__device__ __forceinline__ unsigned smem_u32(const void *p) { return (unsigned)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(unsigned bar, unsigned count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;\n" :: "r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(unsigned bar, unsigned bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;\n" :: "r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(unsigned bar, unsigned parity) {
  asm volatile("{\n .reg .pred P1;\n LAB_WAIT:\n mbarrier.try_wait.parity.shared::cta.b64 P1, [%0], %1;\n @P1 bra DONE;\n bra LAB_WAIT;\n DONE:\n }\n"
               :: "r"(bar), "r"(parity) : "memory");
}
__device__ __forceinline__ unsigned mapa_u32(unsigned addr, unsigned rank) {
  unsigned r;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;\n" : "=r"(r) : "r"(addr), "r"(rank));
  return r;
}
__device__ __forceinline__ void st_async_f64(unsigned remote_addr, double v, unsigned remote_bar) {
  asm volatile("st.async.weak.shared::cluster.mbarrier::complete_tx::bytes.b64 [%0], %1, [%2];\n"
               :: "r"(remote_addr), "l"(__double_as_longlong(v)), "r"(remote_bar) : "memory");
}

template <bool BACKWARD, int CL>
__device__ __forceinline__ void
dense_solve_body(int m, const double *L, const double *dinv, const int *perm, const double *b, double *yout,
                 const double *dscale, const int *flag, const double *lb, int nb, unsigned long long *tdbg) {
  extern __shared__ double smem[];
  double *ys = smem;                                    // m doubles (rounded up to even)
  double *ring = smem + ((m + 1) & ~1);                 // SOLVE_WARPS x 2 x 1024 doubles
  volatile int *ready = (volatile int *)(ring + SOLVE_WARPS * 2 * PB * PB);
  unsigned long long *bars = (unsigned long long *)(ring + SOLVE_WARPS * 2 * PB * PB + ((nb + 1) >> 1));   // one mbarrier per block row
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  namespace cg = cooperative_groups;
  unsigned crank = 0;
  if (CL > 1) crank = cg::this_cluster().block_rank();
  const int rhs = blockIdx.x / CL;
  const double *bb = b + (long long)rhs * m;
  double *yy = yout + (long long)rhs * m;
  const int ld = m;
  double *myring = ring + warp * 2 * PB * PB;
  auto gtime = [] { unsigned long long t; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t)); return t; };
  if (tdbg && threadIdx.x == 0 && blockIdx.x == 0) tdbg[nb] = gtime();
  for (int i = threadIdx.x; i < nb; i += blockDim.x) {
    ready[i] = 0;
    if (CL > 1) {                                       // block row i arrives as min(PB, m - i*PB) doubles from its owner
      mbar_init(smem_u32(bars + i), 1);
      asm volatile("fence.mbarrier_init.release.cluster;\n" ::: "memory");
      mbar_expect_tx(smem_u32(bars + i), 8u * (unsigned)min(PB, m - i * PB));
    }
  }
  __syncthreads();
  if (CL > 1) cg::this_cluster().sync();                // nobody signals a remote barrier before it is armed
  if (tdbg && threadIdx.x == 0 && blockIdx.x == 0) tdbg[nb + 1] = gtime();
  for (int step = warp * CL + (int)crank; step < nb; step += SOLVE_WARPS * CL) {
    const int br = BACKWARD ? (nb - 1 - step) : step;
    const int k0 = br * PB, w = min(PB, m - k0);
    const int nprev = step;                              // number of solved blocks this row depends on
    // element (row k0+lane, column of block j) -> ring slot [c][lane]; rows beyond the matrix are not fetched
    auto fetch = [&](int t) {                            // t-th dependency in solve order
      if (t < nprev && lane < w) {
        const int j = BACKWARD ? (nb - 1 - t) : t;
        const double *Lp = L + (long long)(j * PB) * ld + k0 + lane;
        double *dst = myring + (t & 1) * PB * PB + lane;
        const int wj = min(PB, m - j * PB);
        for (int c = 0; c < wj; c++) cp_async8(dst + c * PB, Lp + (long long)c * ld);
      }
      cp_async_commit();
    };
    fetch(0); fetch(1);
    const double *Di = dinv + (long long)br * PB * PB;
    double di[PB];
#pragma unroll
    for (int c = 0; c < PB; c++) di[c] = BACKWARD ? Di[lane * PB + c] : Di[c * PB + lane];
    double acc0 = 0.0, acc1 = 0.0, acc2 = 0.0, acc3 = 0.0;
    // everything the epilogue needs from global memory is fetched now, off the dependent chain
    int pk = 0;
    double dk = 1.0;
    if (lane < w) {
      pk = perm[k0 + lane];
      acc0 = BACKWARD ? bb[k0 + lane] : bb[pk];
      if (!BACKWARD && dscale) {                          // ./d with deninfac's repair of skipped pivots
        dk = dscale[k0 + lane];
        if (flag && flag[k0 + lane] == 1 && dk <= lb[k0 + lane]) dk = 1.0;
      }
    }
    for (int t = 0; t < nprev; t++) {
      const int j = BACKWARD ? (nb - 1 - t) : t;
      cp_async_wait<1>();                                // group t has landed (only t+1 may be in flight)
      if (CL > 1) mbar_wait(smem_u32(bars + j), 0);       // y_j has been delivered into this CTA's shared memory
      else {
        while (ready[j] == 0) { __nanosleep(20); }        // back off: spinning warps starve the shared-memory pipe
        __threadfence_block();
      }
      __syncwarp();
      const volatile double *yv = ys + j * PB;
      const double *lv = myring + (t & 1) * PB * PB + lane;
      const int wj = min(PB, m - j * PB);
      if (lane < w) {
        if (wj == PB) {
#pragma unroll
          for (int c = 0; c < PB; c += 4) {
            acc0 -= lv[c * PB] * yv[c];
            acc1 -= lv[(c + 1) * PB] * yv[c + 1];
            acc2 -= lv[(c + 2) * PB] * yv[c + 2];
            acc3 -= lv[(c + 3) * PB] * yv[c + 3];
          }
        } else {
          for (int c = 0; c < wj; c++) acc0 -= lv[c * PB] * yv[c];
        }
      }
      __syncwarp();                                      // everyone is done with slot t&1
      fetch(t + 2);
    }
    cp_async_wait<0>();
    const double acc = (acc0 + acc1) + (acc2 + acc3);
    // diagonal block: y = inv(L11) s  (forward)  or  y = inv(L11)' s  (backward)
    double y0 = 0.0, y1 = 0.0, y2 = 0.0, y3 = 0.0;
#pragma unroll
    for (int c = 0; c < PB; c += 4) {
      y0 += di[c] * __shfl_sync(0xffffffffu, acc, c);
      y1 += di[c + 1] * __shfl_sync(0xffffffffu, acc, c + 1);
      y2 += di[c + 2] * __shfl_sync(0xffffffffu, acc, c + 2);
      y3 += di[c + 3] * __shfl_sync(0xffffffffu, acc, c + 3);
    }
    const double yv = (y0 + y1) + (y2 + y3);
    if (lane < w) {
      if (CL > 1) {
        const unsigned ya = smem_u32(ys + k0 + lane), ba = smem_u32(bars + br);
#pragma unroll
        for (int r = 0; r < CL; r++) st_async_f64(mapa_u32(ya, (unsigned)r), yv, mapa_u32(ba, (unsigned)r));
      } else ys[k0 + lane] = yv;
    }
    if (CL > 1) {
      __syncwarp();
    } else {
      __threadfence_block();
      __syncwarp();
      if (lane == 0) ready[br] = 1;
    }
    if (tdbg && lane == 0 && blockIdx.x < CL) tdbg[br] = gtime();
    if (lane < w) {                                       // the result leaves after the consumers have been released
      if (!BACKWARD) yy[k0 + lane] = dscale ? yv / dk : yv;
      else yy[pk] = yv;
    }
  }
  if (CL > 1) cg::this_cluster().sync();                // no CTA may exit while peers still write into its shared memory
  if (tdbg && threadIdx.x == 0 && blockIdx.x == 0) tdbg[nb + 2] = gtime();
}

template <bool BACKWARD>
__global__ void __launch_bounds__(SOLVE_WARPS * 32)
dense_solve_kernel(int m, const double *L, const double *dinv, const int *perm, const double *b, double *yout,
                   const double *dscale, const int *flag, const double *lb, int nb, unsigned long long *tdbg) {
  dense_solve_body<BACKWARD, 1>(m, L, dinv, perm, b, yout, dscale, flag, lb, nb, tdbg);
}
template <bool BACKWARD>
__global__ void __cluster_dims__(SOLVE_CLUSTER, 1, 1) __launch_bounds__(SOLVE_WARPS * 32)
dense_solve_cluster_kernel(int m, const double *L, const double *dinv, const int *perm, const double *b, double *yout,
                           const double *dscale, const int *flag, const double *lb, int nb, unsigned long long *tdbg) {
  dense_solve_body<BACKWARD, SOLVE_CLUSTER>(m, L, dinv, perm, b, yout, dscale, flag, lb, nb, tdbg);
}

// ---------------------------------------------------------------------------------- host side
static __global__ void dense_permuteP_kernel(int m, const int *perm, const int *Xjc, const int *Xir, const double *Xpr,
                                             double *W, double *diagX) {
  const int j = blockIdx.x;
  const int pj = perm[j];
  const int b0 = Xjc[pj], b1 = Xjc[pj + 1];
  const bool dense = (b1 - b0) == m;
  double *col = W + (long long)j * m;
  for (int t = threadIdx.x; t < m; t += blockDim.x) {
    double v = 0.0;
    if (t >= j) {
      const int pi = perm[t];
      if (dense) v = Xpr[b0 + pi];
      else {
        int lo = b0, hi = b1;
        while (lo < hi) { int mid = (lo + hi) >> 1; if (Xir[mid] < pi) lo = mid + 1; else hi = mid; }
        if (lo < b1 && Xir[lo] == pi) v = Xpr[lo];
      }
      if (t == j) diagX[j] = v;
    }
    col[t] = v;
  }
}

int dense_make_transpose(sb200_chol_plan *pl, const double *rect);

int dense_factor_prepare(sb200_chol_plan *pl) {
  const int m = pl->m;
  pl->npanels = (m + PB - 1) / PB;
  SB_TRY(pl->d_work.alloc((size_t)m * m));
  SB_TRY(pl->d_dinv.alloc((size_t)pl->npanels * PB * PB));
  SB_TRY(pl->d_bar.alloc(4 + (size_t)pl->npanels + 1));
  return 0;
}

// Xpr_dev -> W (plan scratch) is done by the caller through dense_permuteP; here: bounds + factor.
int dense_factor(sb200_chol_plan *pl, const double *Xpr, const double *absd, sb200_chol_pars pars,
                 double *rect, double *d, int *flag, double *sval, void (*bounds)(sb200_chol_plan *, const double *, sb200_chol_pars)) {
  cudaStream_t st = ctx().stream;
  const int m = pl->m;
  dense_permuteP_kernel<<<m, 256, 0, st>>>(m, pl->d_perm.p, pl->d_Xjc.p, pl->d_Xir.p, Xpr, pl->d_work.p, pl->d_diagX.p);
  SB_LAUNCH_CHECK_N("dense_permuteP_kernel");
  bounds(pl, absd, pars);
  SB_CUDA(cudaMemsetAsync(pl->d_bar.p, 0, sizeof(unsigned) * (4 + pl->npanels + 1), st));
  // cooperative launch: every CTA must be resident
  int per_sm = 0;
  SB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, dense_ldl_kernel, 256, 0));
  SB_CHECK(per_sm >= 1, "dense_ldl_kernel cannot be resident");
  const int nslab = (std::max(m - PB, 0) + TS - 1) / TS;
  int want = nslab > 0 ? nslab * (nslab + 1) / 2 + 1 : 1;      // the tiles of the first panel + the panel CTA
  int grid = std::min(want, per_sm * ctx().sm_count);
  double *W = pl->d_work.p, *dinv = pl->d_dinv.p, *lb = pl->d_lb.p, *scal = pl->d_scal.p, *diagX = pl->d_diagX.p, *vs = pl->d_vscratch.p;
  unsigned *bar = pl->d_bar.p;
  int mm = m;
  double maxu = pars.maxu;
  static long long *s_tdbg = nullptr;
  long long *tdbg = nullptr;
  if (getenv("SB200_CHOL_TIMING")) {
    if (!s_tdbg) cudaMalloc((void **)&s_tdbg, sizeof(long long) * 8 * 4096);
    tdbg = s_tdbg;
  }
  void *args[] = {&mm, &W, &rect, &d, &lb, &scal, &maxu, &flag, &sval, &diagX, &vs, &dinv, &bar, &tdbg};
  SB_CUDA(cudaLaunchCooperativeKernel((void *)dense_ldl_kernel, dim3(grid), dim3(256), args, 0, st));
  SB_LAUNCH_CHECK_N("dense_ldl_kernel");
  if (tdbg) {
    std::vector<long long> h(8 * pl->npanels);
    cudaStreamSynchronize(st);
    cudaMemcpy(h.data(), tdbg, sizeof(long long) * h.size(), cudaMemcpyDeviceToHost);
    // probes of CTA 0 (the panel CTA): [4] start of phase B(p), [1] look-ahead starts, [2] (slot of panel p+1)
    // its factorisation is done, [5] published, [6] grid barrier passed
    double prep = 0, fac = 0, pub = 0, bar = 0;
    for (int p = 0; p + 1 < pl->npanels; p++) {
      const long long *t = h.data() + 8 * p;
      prep += t[1] - t[4]; fac += t[8 + 2] - t[1]; pub += t[5] - t[8 + 2]; bar += t[6] - t[5];
    }
    fprintf(stderr, "[dense_ldl timing, panel CTA clocks summed over %d panels] first panel %.0f  load L11 %.0f  form+factor next block %.0f  publish %.0f  barrier %.0f  (total %.0f)\n",
            pl->npanels, (double)(h[3] - h[0]), prep, fac, pub, bar, (double)(h[8 * (pl->npanels - 1) + 6] - h[0]));
  }
  return dense_make_transpose(pl, rect);                 // the working copy is dead now: reuse it for L'
}

// Lt = L' (lower triangle of L mirrored into the upper triangle of a second array) so that the
// backward solve streams it with the same coalesced pattern as the forward solve.
static __global__ void dense_transpose_kernel(int m, const double *L, double *Lt) {
  __shared__ double tile[32][33];
  const int bi = blockIdx.x, bj = blockIdx.y;            // tile (rows bi, cols bj) of L, bi >= bj
  if (bi < bj) return;
  const int r0 = bi * 32, c0 = bj * 32;
  for (int jj = threadIdx.y; jj < 32; jj += blockDim.y) {
    const int r = r0 + threadIdx.x, c = c0 + jj;
    tile[jj][threadIdx.x] = (r < m && c < m && r > c) ? L[(long long)c * m + r] : 0.0;
  }
  __syncthreads();
  for (int jj = threadIdx.y; jj < 32; jj += blockDim.y) {
    const int c = c0 + threadIdx.x, r = r0 + jj;         // Lt(c, r) = L(r, c)
    if (c < m && r < m) Lt[(long long)r * m + c] = tile[threadIdx.x][jj];
  }
}
int dense_make_transpose(sb200_chol_plan *pl, const double *rect) {
  const int nb = (pl->m + 31) / 32;
  dense_transpose_kernel<<<dim3(nb, nb), dim3(32, 8), 0, ctx().stream>>>(pl->m, rect, pl->d_work.p);
  SB_LAUNCH_CHECK_N("dense_transpose_kernel");
  return 0;
}

static int solve_launch(bool backward, sb200_chol_plan *pl, const double *rect, const double *b, double *y, int nrhs,
                        const double *dscale, const int *flag) {
  const int m = pl->m, nb = (m + PB - 1) / PB;
  size_t shm = sizeof(double) * (((m + 1) & ~1) + SOLVE_WARPS * 2 * PB * PB + ((nb + 1) >> 1) + nb);      // y, rings, flags, mbarriers
  SB_CHECK(shm <= 200 * 1024, "dense solve: m=%d too large for the shared-memory dataflow kernel", m);
  cudaStream_t st = ctx().stream;
  static const bool use_cluster = !(getenv("SB200_SOLVE_CLUSTER") && atoi(getenv("SB200_SOLVE_CLUSTER")) == 0);
  static unsigned long long *s_tdbg = nullptr;
  unsigned long long *tdbg = nullptr;
  if (getenv("SB200_SOLVE_TIMING")) {
    if (!s_tdbg) cudaMalloc((void **)&s_tdbg, sizeof(unsigned long long) * 8192);
    tdbg = s_tdbg;
    cudaMemsetAsync(tdbg, 0, sizeof(unsigned long long) * 8192, st);
  }
  // a cluster only pays when there are block rows for more than one CTA's warps to overlap
  const bool cl = use_cluster && nb > 2;
  if (backward) {
    if (cl) {
      if (shm > 48 * 1024) SB_CUDA(cudaFuncSetAttribute(dense_solve_cluster_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)shm));
      dense_solve_cluster_kernel<true><<<nrhs * SOLVE_CLUSTER, SOLVE_WARPS * 32, shm, st>>>(m, pl->d_work.p, pl->d_dinv.p, pl->d_perm.p, b, y, nullptr, nullptr, nullptr, nb, tdbg);
    } else {
      if (shm > 48 * 1024) SB_CUDA(cudaFuncSetAttribute(dense_solve_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)shm));
      dense_solve_kernel<true><<<nrhs, SOLVE_WARPS * 32, shm, st>>>(m, pl->d_work.p, pl->d_dinv.p, pl->d_perm.p, b, y, nullptr, nullptr, nullptr, nb, tdbg);
    }
  } else {
    if (cl) {
      if (shm > 48 * 1024) SB_CUDA(cudaFuncSetAttribute(dense_solve_cluster_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)shm));
      dense_solve_cluster_kernel<false><<<nrhs * SOLVE_CLUSTER, SOLVE_WARPS * 32, shm, st>>>(m, rect, pl->d_dinv.p, pl->d_perm.p, b, y, dscale, flag, pl->d_lb.p, nb, tdbg);
    } else {
      if (shm > 48 * 1024) SB_CUDA(cudaFuncSetAttribute(dense_solve_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)shm));
      dense_solve_kernel<false><<<nrhs, SOLVE_WARPS * 32, shm, st>>>(m, rect, pl->d_dinv.p, pl->d_perm.p, b, y, dscale, flag, pl->d_lb.p, nb, tdbg);
    }
  }
  SB_LAUNCH_CHECK_N(backward ? "dense_solve_kernel<bw>" : "dense_solve_kernel<fw>");
  if (tdbg) {
    std::vector<unsigned long long> h(nb + 3);
    cudaStreamSynchronize(st);
    cudaMemcpy(h.data(), tdbg, sizeof(unsigned long long) * h.size(), cudaMemcpyDeviceToHost);
    fprintf(stderr, "[dense_solve %s timing, ns from kernel start] init+cluster sync %llu  rows:", backward ? "bw" : "fw", h[nb + 1] - h[nb]);
    for (int i = 0; i < nb; i++) { const int br = backward ? nb - 1 - i : i; fprintf(stderr, " %lld", (long long)(h[br] - h[nb])); }
    fprintf(stderr, "  end %llu\n", h[nb + 2] - h[nb]);
  }
  return 0;
}
int dense_fwsolve(sb200_chol_plan *pl, const double *rect, const double *b, double *y, int nrhs, const double *dscale, const int *flag) {
  return solve_launch(false, pl, rect, b, y, nrhs, dscale, flag);
}
int dense_bwsolve(sb200_chol_plan *pl, const double *rect, const double *b, double *y, int nrhs) {
  return solve_launch(true, pl, rect, b, y, nrhs, nullptr, nullptr);
}

// inverses of the diagonal blocks from an L that did not come from dense_factor (MEX-level solves)
static __global__ void dense_dinv_kernel(int m, const double *Lo, double *dinv) {
  __shared__ double A[PB][PB + 1];
  const int pi = blockIdx.x, p0 = pi * PB, w = min(PB, m - p0), lane = threadIdx.x;
  for (int idx = lane; idx < PB * PB; idx += 32) {
    int r = idx % PB, c = idx / PB;
    A[r][c] = (r < w && c < w && r > c) ? Lo[(long long)(p0 + c) * m + p0 + r] : 0.0;
  }
  __syncwarp();
  double x[PB];
#pragma unroll
  for (int i = 0; i < PB; i++) x[i] = (i == lane) ? 1.0 : 0.0;
#pragma unroll
  for (int i = 1; i < PB; i++) {
    double acc = 0.0;
#pragma unroll
    for (int j = 0; j < PB; j++) if (j < i) acc += A[i][j] * x[j];
    x[i] -= acc;
  }
  double *out = dinv + (long long)pi * PB * PB + lane * PB;
#pragma unroll
  for (int i = 0; i < PB; i++) out[i] = x[i];
}
int dense_compute_dinv(sb200_chol_plan *pl, const double *rect) {
  dense_dinv_kernel<<<pl->npanels, 32, 0, ctx().stream>>>(pl->m, rect, pl->d_dinv.p);
  SB_LAUNCH_CHECK_N("dense_dinv_kernel");
  return dense_make_transpose(pl, rect);
}

}  // namespace sb
