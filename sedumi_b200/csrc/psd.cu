// psd.cu -- per-PSD-block dense algebra: invcholfac (D = U'U) and psdscale (Y = T'XT).
//
// Reference semantics:
//   invcholfac.c:122-141  per block: Z = triu(U)'*triu(U) (utmulx, triuaux.c:175-186),
//                         symmetrised, then Y(perm,perm) = Z (invmatperm, triuaux.c:61-72)
//   psdscale.m:76-110     per block: T = tril(U) (transp=0) or triu(U) (transp=1) of the
//                         stored n x n array, X optionally X(perm,perm) before (transp=0)
//                         or the result scattered to (perm,perm) after (transp=1); Y = T'*X*T
//
// GPU design: every block is a set of 64x64 tiles in ONE batched launch of the DMMA tile
// GEMM (gemm.cuh).  Both operations are written as "NT" products over Tt = T' so that all
// tile loads are contiguous:
//   invcholfac:  Z(i,j)  = sum_k Tt(i,k) Tt(j,k)            (Tt = triu(U)', lower triangular)
//   psdscale:    Wt(c,i) = sum_k Tt(c,k) X(i,k);  Y(i,c) = sum_k Tt(i,k) Wt(c,k)
// and the triangular k-ranges are skipped per tile.  Descriptors and tile lists depend only
// on K.s, so they live in a cached plan; per call only the block data moves.
#include <map>
#include "gemm.cuh"
#include "sb_internal.h"

struct sb200_psd_plan {
  int nblk = 0;
  long long lenud = 0, sumn = 0;
  int maxn = 0;
  std::vector<int> n;
  std::vector<long long> off;      // offset of block k in a lenud vector
  std::vector<int> poff;           // offset of block k in a perm vector
  // device
  sb::DevBuf<int> d_n, d_poff;
  sb::DevBuf<long long> d_off;
  sb::DevBuf<sb::GemmDesc> d_desc_ichol, d_desc_s1_lo, d_desc_s1_up, d_desc_s2_lo, d_desc_s2_up, d_desc_full, d_desc_lower;
  sb::DevBuf<int> d_qcol_blk, d_qcol_j0;     // column groups for the Householder accumulation
  int nqgroups = 0;
  sb::DevBuf<sb::GemmTile> d_tiles_full, d_tiles_lower;
  int ntiles_full = 0, ntiles_lower = 0;
  // blocked (compact WY) Householder accumulation for large blocks: step s handles panel P_k-1-s of
  // every block that still has one; three GEMM launches per step
  bool wy = false;            // GEMM-based WY (blocks too large for wy_rows_kernel's shared memory)
  bool wy_rows = false;       // wy_rows_kernel
  size_t wy_rows_smem = 0;
  int wy_steps = 0, wy_npanels = 0;
  struct WyStep { int d1, d2, d3; int t1, n1, t2, n2, t3, n3; };   // descriptor / tile ranges per step
  std::vector<WyStep> wy_sched;
  sb::DevBuf<sb::GemmDesc> d_wy_desc;
  sb::DevBuf<sb::GemmTile> d_wy_tiles;
  sb::DevBuf<int> d_wy_pblk, d_wy_pidx;          // per panel: block, panel index
  sb::DevBuf<long long> d_wy_toff;               // per block: offset of its first T (32x32 each)
  sb::DevBuf<double> d_wy_T, d_wy_Y, d_wy_Y2, d_wy_G;
  int wyb = 32;                                     // reflectors per panel: 32 (row kernel) or 128 (GEMM path)
  int wy_gd = 0, wy_gt = 0, wy_gn = 0;              // descriptors / tiles of the Gram products V_p' V_p (GEMM path)
  // workspaces (lenud doubles each)
  sb::DevBuf<double> d_Tt, d_Wt, d_Xp, d_Y;
  sb::DevBuf<int> d_perm;
};

namespace sb {

// blockIdx.y = PSD block; Tt(c,k) = mask ? U[k + c*n] : 0 with mask (k<=c) for upper=1, (k>=c) for upper=0
__global__ void tri_transpose_kernel(const int *ns, const long long *offs, const double *u, double *Tt, int upper) {
  const int n = ns[blockIdx.y];
  const double *U = u + offs[blockIdx.y];
  double *T = Tt + offs[blockIdx.y];
  __shared__ double tile[32][33];
  const int tilesPerDim = (n + 31) / 32;
  for (int t = blockIdx.x; t < tilesPerDim * tilesPerDim; t += gridDim.x) {
    int k0 = (t % tilesPerDim) * 32, c0 = (t / tilesPerDim) * 32;
    for (int j = threadIdx.y; j < 32; j += blockDim.y) {
      int k = k0 + threadIdx.x, c = c0 + j;
      tile[j][threadIdx.x] = (k < n && c < n) ? U[k + (long long)c * n] : 0.0;
    }
    __syncthreads();
    for (int j = threadIdx.y; j < 32; j += blockDim.y) {
      int c = c0 + threadIdx.x, k = k0 + j;
      if (c < n && k < n) {
        bool keep = upper ? (k <= c) : (k >= c);
        T[c + (long long)k * n] = keep ? tile[threadIdx.x][j] : 0.0;
      }
    }
    __syncthreads();
  }
}

// The same for blocks up to PERM_COLS_MAXN, without the symmetric read: one warp per column, the column passes through
// shared memory so that both the global read and the global write are contiguous (perm_block_kernel gathers or scatters
// 8-byte words at random inside a column: 1.9 TB/s on the 64 x 200 problem, 14 launches per iteration).
//   gather : out(i, j)       = in(p[i], p[j])    -> read column p[j],  out(i, j)    = col[p[i]]
//   scatter: out(p[i], p[j]) = in(i, j)          -> read column j,     out(r, p[j]) = col[pinv[r]]
static const int PERM_COLS_MAXN = 512, PERM_COLS_W = 8;
__global__ void __launch_bounds__(32 * PERM_COLS_W)
perm_cols_kernel(const int *ns, const long long *offs, const int *poffs, const int *perm, const double *in, double *out, int gather) {
  extern __shared__ double pc_sm[];
  const int n = ns[blockIdx.y];
  if ((int)blockIdx.x * PERM_COLS_W >= n) return;
  const long long off = offs[blockIdx.y];
  const int *p = perm + poffs[blockIdx.y];
  double *cols = pc_sm;                                   // [PERM_COLS_W][n]
  int *sp = (int *)(pc_sm + (size_t)PERM_COLS_W * n);     // p (gather) or its inverse (scatter)
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    const int pi = p[i];
    if (gather) sp[i] = pi; else sp[pi] = i;
  }
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int j = blockIdx.x * PERM_COLS_W + warp;
  double *col = cols + (size_t)warp * n;
  int pj = 0;
  if (j < n) {
    pj = p[j];
    const double *src = in + off + (long long)(gather ? pj : j) * n;
    for (int i = lane; i < n; i += 32) col[i] = src[i];
  }
  __syncthreads();
  if (j < n) {
    double *dst = out + off + (long long)(gather ? j : pj) * n;
    for (int i = lane; i < n; i += 32) dst[i] = col[sp[i]];
  }
}

// out(i,j) = in(p[i], p[j])  (gather=1)   or   out(p[i], p[j]) = in(i,j)  (gather=0); sym=1 reads in(max,min)
__global__ void perm_block_kernel(const int *ns, const long long *offs, const int *poffs, const int *perm,
                                  const double *in, double *out, int gather, int sym) {
  const int n = ns[blockIdx.y];
  const long long off = offs[blockIdx.y];
  const int *p = perm ? perm + poffs[blockIdx.y] : nullptr;
  const long long tot = (long long)n * n;
  for (long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x; idx < tot; idx += (long long)gridDim.x * blockDim.x) {
    int i = (int)(idx % n), j = (int)(idx / n);
    int pi = p ? p[i] : i, pj = p ? p[j] : j;
    if (gather) out[off + idx] = in[off + pi + (long long)pj * n];
    else {
      double v = sym ? in[off + max(i, j) + (long long)min(i, j) * n] : in[off + idx];
      out[off + pi + (long long)pj * n] = v;
    }
  }
}


// ---------------------------------------------------------------- Householder frames (psdframeit / psdinvjmul)
// frms block k: n x n, column c (c < n-1) holds reflector vector c_c in rows c..n-1, last column holds
// beta_0..beta_{n-2};  H_c = I - c_c c_c'/beta_c ;  Qb = H_0 H_1 ... H_{n-2}   (reflect.c:203-215, qrK.c:86-122).
// Column j of Qb is H_0...H_{min(j,n-2)} e_j and columns are independent: one warp per column,
// 8 columns per CTA, the reflectors streamed from L2.  Q is written column-major.
__global__ void __launch_bounds__(256)
householder_q_kernel(const int *grp_blk, const int *grp_j0, const int *ns, const long long *offs,
                     const double *frms, double *Q) {
  const int k = grp_blk[blockIdx.x];
  const int n = ns[k];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int j = grp_j0[blockIdx.x] + warp;
  if (j >= n) return;
  const double *F = frms + offs[k];
  const double *beta = F + (long long)n * n - n;
  double *q = Q + offs[k] + (long long)j * n;
  if (n <= 96) {
    // the column lives in registers (rows lane, lane+32, lane+64); the next reflector is fetched while the
    // dot product of the current one is reduced
    double q0 = (lane == j) ? 1.0 : 0.0, q1 = (lane + 32 == j) ? 1.0 : 0.0, q2 = (lane + 64 == j) ? 1.0 : 0.0;
    int c = min(j, n - 2);
    auto ld = [&](int cc, int r) { return (cc >= 0 && r >= cc && r < n) ? F[(long long)cc * n + r] : 0.0; };
    double v0 = ld(c, lane), v1 = ld(c, lane + 32), v2 = ld(c, lane + 64);
    double bc = c >= 0 ? beta[c] : 1.0;
    for (; c >= 0; c--) {
      const double w0 = ld(c - 1, lane), w1 = ld(c - 1, lane + 32), w2 = ld(c - 1, lane + 64);
      const double bn = c >= 1 ? beta[c - 1] : 1.0;
      double t = v0 * q0 + v1 * q1 + v2 * q2;
      for (int o = 16; o > 0; o >>= 1) t += __shfl_xor_sync(0xffffffffu, t, o);
      const double a = t / (-bc);                       // elqxq is called with -beta (reflect.c:214)
      q0 += a * v0; q1 += a * v1; q2 += a * v2;
      v0 = w0; v1 = w1; v2 = w2; bc = bn;
    }
    if (lane < n) q[lane] = q0;
    if (lane + 32 < n) q[lane + 32] = q1;
    if (lane + 64 < n) q[lane + 64] = q2;
    return;
  }
  for (int i = lane; i < n; i += 32) q[i] = (i == j) ? 1.0 : 0.0;
  __syncwarp();
  for (int c = min(j, n - 2); c >= 0; c--) {
    const double *v = F + (long long)c * n;           // v[i], i = c..n-1
    double t = 0.0;
    for (int i = c + lane; i < n; i += 32) t += v[i] * q[i];
    for (int o = 16; o > 0; o >>= 1) t += __shfl_xor_sync(0xffffffffu, t, o);
    const double a = t / (-beta[c]);                  // elqxq is called with -beta (reflect.c:214)
    for (int i = c + lane; i < n; i += 32) q[i] += a * v[i];
    __syncwarp();
  }
}

// ---- compact-WY pieces (blocks too large for the one-warp-per-column kernel above).
// T_p^{-1} = striu(V_p' V_p) + diag(beta_p) for panel p (32 reflectors) of a block; exact for any beta:
// (I - V T V')(I - v v'/b) = I - [V v] [[T, -T V'v/b],[0, 1/b]] [V v]'.   One CTA per (block, panel).
static const int WYB = 32;
__global__ void __launch_bounds__(256)
wy_t_kernel(const int *pblk, const int *pidx, const int *ns, const long long *offs, const long long *toff,
            const double *frms, double *Tall) {
  const int k = pblk[blockIdx.x], p = pidx[blockIdx.x];
  const int n = ns[k];
  const double *F = frms + offs[k];
  const double *beta = F + (long long)n * n - n;
  const int c0 = p * WYB, bp = min(WYB, n - 1 - c0);
  __shared__ double U[WYB][WYB + 1];
  __shared__ double Vc[32][WYB + 1];                 // a chunk of 32 rows of the panel
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  // G = V'V as a small SYRK: rows streamed in chunks of 32 through shared memory, thread (ta,tb) owns the 2x2
  // block G(2ta..2ta+1, 2tb..2tb+1); entries of V above a reflector's own diagonal are structural zeros
  const int ta = threadIdx.x >> 4, tb = threadIdx.x & 15;
  double g00 = 0.0, g01 = 0.0, g10 = 0.0, g11 = 0.0;
  for (int r0 = c0; r0 < n; r0 += 32) {
    for (int idx = threadIdx.x; idx < 32 * WYB; idx += blockDim.x) {
      const int rr = idx & 31, cc = idx >> 5, r = r0 + rr;
      Vc[rr][cc] = (cc < bp && r < n && r >= c0 + cc) ? F[(long long)(c0 + cc) * n + r] : 0.0;
    }
    __syncthreads();
#pragma unroll 8
    for (int rr = 0; rr < 32; rr++) {
      const double a0 = Vc[rr][2 * ta], a1 = Vc[rr][2 * ta + 1], b0 = Vc[rr][2 * tb], b1 = Vc[rr][2 * tb + 1];
      g00 += a0 * b0; g01 += a0 * b1; g10 += a1 * b0; g11 += a1 * b1;
    }
    __syncthreads();
  }
  // T^{-1} = striu(G) + diag(beta)
  {
    const int i0 = 2 * ta, j0 = 2 * tb;
    U[i0][j0] = (i0 < j0) ? g00 : 0.0; U[i0][j0 + 1] = (i0 < j0 + 1) ? g01 : 0.0;
    U[i0 + 1][j0] = (i0 + 1 < j0) ? g10 : 0.0; U[i0 + 1][j0 + 1] = (i0 + 1 < j0 + 1) ? g11 : 0.0;
  }
  __syncthreads();
  if (threadIdx.x < WYB) U[threadIdx.x][threadIdx.x] = threadIdx.x < bp ? beta[c0 + threadIdx.x] : 1.0;
  __syncthreads();
  // T = inv(U), U upper triangular: lane j solves U t = e_j from the bottom up
  double *T = Tall + (toff[k] + p) * WYB * WYB;
  if (warp == 0) {
    const int j = lane;
    double t[WYB];
#pragma unroll
    for (int i = 0; i < WYB; i++) t[i] = 0.0;
    if (j < bp) {
#pragma unroll
      for (int i = WYB - 1; i >= 0; i--) {
        if (i < bp && i <= j) {
          double acc = (i == j) ? 1.0 : 0.0;
#pragma unroll
          for (int q = 0; q < WYB; q++) if (q > i && q <= j) acc -= U[i][q] * t[q];
          t[i] = acc / U[i][i];
        }
      }
    }
#pragma unroll
    for (int i = 0; i < WYB; i++) T[i + j * WYB] = t[i];     // column-major 32x32, zero padded
  }
}

// Wide panels (GEMM path, WYBIG reflectors): G = V_p' V_p comes from the tile-GEMM engine; this kernel forms
// U = striu(G) + diag(beta_p) in shared memory and inverts it, one thread per column of T = inv(U) (back substitution).
static const int WYBIG = 128;
__global__ void __launch_bounds__(WYBIG)
wy_tinv_big_kernel(const int *pblk, const int *pidx, const int *ns, const long long *offs, const long long *toff,
                   const double *frms, const double *Gall, double *Tall) {
  extern __shared__ double Ubig[];                   // WYBIG x (WYBIG + 1)
  const int k = pblk[blockIdx.x], p = pidx[blockIdx.x];
  const int n = ns[k];
  const double *beta = frms + offs[k] + (long long)n * n - n;
  const int c0 = p * WYBIG, bp = min(WYBIG, n - 1 - c0);
  const double *G = Gall + (toff[k] + p) * WYBIG * WYBIG;
  double *T = Tall + (toff[k] + p) * WYBIG * WYBIG;
  const int j = threadIdx.x, ldu = WYBIG + 1;
  for (int i = 0; i < WYBIG; i++)                    // column j of U (coalesced over j)
    Ubig[i * ldu + j] = (i < bp && j < bp) ? (i < j ? G[i + (long long)j * WYBIG] : (i == j ? beta[c0 + i] : 0.0)) : (i == j ? 1.0 : 0.0);
  __syncthreads();
  // U t = e_j from the bottom up; t is written straight into T(:, j) and read back from there (own column only)
  double *t = T + (long long)j * WYBIG;
  for (int i = WYBIG - 1; i >= 0; i--) {
    double acc = 0.0;
    if (j < bp && i <= j) {
      acc = (i == j) ? 1.0 : 0.0;
      for (int q = i + 1; q <= j; q++) acc -= Ubig[i * ldu + q] * t[q];
      acc /= Ubig[i * ldu + i];
    }
    t[i] = acc;
  }
}

// Q from the panels' T factors, eight columns of Q per CTA.  Row i of R = Q' evolves independently of the
// others:  r <- r - ((r V_p) T_p') V_p'  for p = last..0, so a CTA keeps its 8 rows of R in shared memory
// and streams each panel V_p (rows c0..n-1, 32 reflectors) twice through a double-buffered cp.async
// ring: once for Y = R V_p, once for R -= (Y T_p') V_p'.  Compared with one warp per column applying the
// reflectors one by one, the 8 columns share every load of V (8x less L2 traffic, which bounded that
// kernel) and the dot/axpy pairs become two small matrix products.
static const int WY_RW = 8, WY_CH = 128;
__global__ void __launch_bounds__(256)
wy_rows_kernel(const int *grp_blk, const int *grp_j0, const int *ns, const long long *offs, const long long *toff,
               const double *frms, const double *Tall, double *Q) {
  extern __shared__ double wy_sm[];
  const int k = grp_blk[blockIdx.x], i0 = grp_j0[blockIdx.x];
  const int n = ns[k];
  const int nld = (n + 1) & ~1;
  double *Rs = wy_sm;                                              // [WY_RW][nld]
  double (*Vs)[WY_CH][WYB + 1] = (double (*)[WY_CH][WYB + 1])(Rs + WY_RW * nld);   // [2][CH][33]
  double *Ys = (double *)(Vs + 2);                                 // [WY_RW][WYB]
  double *Y2s = Ys + WY_RW * WYB;
  double (*Ts)[WYB + 1] = (double (*)[WYB + 1])(Y2s + WY_RW * WYB);
  const double *F = frms + offs[k];
  const int tid = threadIdx.x, ti = tid >> 5, tc = tid & 31;
  for (int idx = tid; idx < WY_RW * nld; idx += blockDim.x) {
    const int i = idx / nld, r = idx % nld;
    Rs[idx] = (r == i0 + i && r < n) ? 1.0 : 0.0;
  }
  const int P = (n - 1 + WYB - 1) / WYB;
  const int pstart = min(P - 1, (min(i0 + WY_RW, n) - 1) / WYB);   // later panels leave these unit rows alone
  for (int p = pstart; p >= 0; p--) {
    const int c0 = p * WYB, bp = min(WYB, n - 1 - c0);
    const int nch = (n - c0 + WY_CH - 1) / WY_CH;
    auto stage = [&](int buf, int r0) {
      const int rr = tid & (WY_CH - 1), r = r0 + rr;
#pragma unroll
      for (int q = 0; q < WYB / 2; q++) {
        const int c = (tid >> 7) + 2 * q;
        const bool valid = (c < bp) && (r < n) && (r >= c0 + c);
        cp_async_8(&Vs[buf][rr][c], valid ? F + r + (long long)(c0 + c) * n : F, valid ? 8 : 0);
      }
      cp_async_commit();
    };
    __syncthreads();                                 // previous panel (or the initialisation) is complete
    const double *T = Tall + (toff[k] + p) * WYB * WYB;
    for (int idx = tid; idx < WYB * WYB; idx += blockDim.x) Ts[idx % WYB][idx / WYB] = T[idx];    // Ts[c][kk] = T(c,kk)
    // ---- Y = R V_p
    double acc = 0.0;
    stage(0, c0);
    for (int ch = 0; ch < nch; ch++) {
      cp_async_wait_all();
      __syncthreads();
      if (ch + 1 < nch) stage((ch + 1) & 1, c0 + (ch + 1) * WY_CH);
      const int r0 = c0 + ch * WY_CH, lim = min(WY_CH, n - r0);
      const double *rrow = Rs + ti * nld + r0;
      const double (*V)[WYB + 1] = Vs[ch & 1];
      double a0 = 0.0, a1 = 0.0, a2 = 0.0, a3 = 0.0;
      int rr = 0;
      for (; rr + 3 < lim; rr += 4) {
        a0 += rrow[rr] * V[rr][tc]; a1 += rrow[rr + 1] * V[rr + 1][tc];
        a2 += rrow[rr + 2] * V[rr + 2][tc]; a3 += rrow[rr + 3] * V[rr + 3][tc];
      }
      for (; rr < lim; rr++) a0 += rrow[rr] * V[rr][tc];
      acc += (a0 + a1) + (a2 + a3);
    }
    Ys[ti * WYB + tc] = acc;
    __syncthreads();
    // ---- Y2 = Y T_p'
    {
      double y2 = 0.0;
#pragma unroll 8
      for (int kk = 0; kk < WYB; kk++) y2 += Ys[ti * WYB + kk] * Ts[tc][kk];
      Y2s[ti * WYB + tc] = y2;
    }
    __syncthreads();
    // ---- R -= Y2 V_p'
    stage(0, c0);
    for (int ch = 0; ch < nch; ch++) {
      cp_async_wait_all();
      __syncthreads();
      if (ch + 1 < nch) stage((ch + 1) & 1, c0 + (ch + 1) * WY_CH);
      const int r0 = c0 + ch * WY_CH;
      const double (*V)[WYB + 1] = Vs[ch & 1];
      const double *y2 = Y2s + ti * WYB;
#pragma unroll
      for (int q = 0; q < WY_CH / 32; q++) {
        const int rr = tc + 32 * q;
        if (r0 + rr < n) {
          double sacc = 0.0;
#pragma unroll 8
          for (int c = 0; c < WYB; c++) sacc += y2[c] * V[rr][c];
          Rs[ti * nld + r0 + rr] -= sacc;
        }
      }
    }
  }
  __syncthreads();
  if (i0 + ti < n) {
    double *q = Q + offs[k] + (long long)(i0 + ti) * n;
    for (int r = tc; r < n; r += 32) q[r] = Rs[ti * nld + r];
  }
}

__global__ void set_identity_kernel(const int *ns, const long long *offs, double *R) {
  const int n = ns[blockIdx.y];
  double *A = R + offs[blockIdx.y];
  const long long tot = (long long)n * n;
  for (long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x; idx < tot; idx += (long long)gridDim.x * blockDim.x)
    A[idx] = (idx % n == idx / n) ? 1.0 : 0.0;
}

// out = transpose(in) per block, optionally scaling row k of the result's k-index:  out(c,k) = in(k,c) * (lab ? lab[k] : 1)
__global__ void transpose_scale_kernel(const int *ns, const long long *offs, const int *poffs, const double *in,
                                       const double *lab, double *out) {
  const int n = ns[blockIdx.y];
  const double *A = in + offs[blockIdx.y];
  double *B = out + offs[blockIdx.y];
  const double *lb = lab ? lab + poffs[blockIdx.y] : nullptr;
  __shared__ double tile[32][33];
  const int tpd = (n + 31) / 32;
  for (int t = blockIdx.x; t < tpd * tpd; t += gridDim.x) {
    int k0 = (t % tpd) * 32, c0 = (t / tpd) * 32;
    for (int jj = threadIdx.y; jj < 32; jj += blockDim.y) {
      int k = k0 + threadIdx.x, c = c0 + jj;
      tile[jj][threadIdx.x] = (k < n && c < n) ? A[k + (long long)c * n] : 0.0;
    }
    __syncthreads();
    for (int jj = threadIdx.y; jj < 32; jj += blockDim.y) {
      int c = c0 + threadIdx.x, k = k0 + jj;
      if (c < n && k < n) B[c + (long long)k * n] = tile[threadIdx.x][jj] * (lb ? lb[k] : 1.0);
    }
    __syncthreads();
  }
}

// mode 0: mirror the lower triangle up (tril2sym); mode 1: out = symmetric matrix built from tril(in);
// mode 2: in-place jdiv on the lower triangle then mirror: m(i,j) *= 2/(x_i+x_j), m(j,j) /= x_j (psdinvjmul.c:69-84)
__global__ void sym_ops_kernel(const int *ns, const long long *offs, const int *poffs, const double *in, double *out,
                               const double *x, int mode) {
  const int n = ns[blockIdx.y];
  const long long off = offs[blockIdx.y];
  const double *xx = x ? x + poffs[blockIdx.y] : nullptr;
  const long long tot = (long long)n * n;
  for (long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x; idx < tot; idx += (long long)gridDim.x * blockDim.x) {
    int i = (int)(idx % n), j = (int)(idx / n);
    if (mode == 1) { out[off + idx] = in[off + max(i, j) + (long long)min(i, j) * n]; continue; }
    if (i < j) continue;                              // the lower-triangle thread owns the pair (i,j),(j,i)
    double v = in[off + i + (long long)j * n];
    if (mode == 2) v = (i == j) ? v / xx[j] : v * (2.0 / (xx[i] + xx[j]));
    out[off + i + (long long)j * n] = v;
    if (i != j) out[off + j + (long long)i * n] = v;
  }
}

// ---------------------------------------------------------------- fused psdscale for small blocks
// One CTA per PSD block, everything in shared memory: T (masked triangle of U), X (optionally
// X(perm,perm)), W = X*T, then Y = T'*W straight to global (optionally scattered to (perm,perm)).
// Replaces 4-5 launches per call by one when max n_k <= PSD_SMALL_MAX (psdscale.m:76-110).
static const int PSD_SMALL_MAX = 96;
static const int PSD_CS = 16;        // output columns per CTA
// Y(:,c) = T' * (X * T(:,c)) is independent per output column c, so a block is split over
// ceil(n/16) CTAs (blockIdx.y) that each keep T and X in shared memory and own 16 columns of W and Y:
// no inter-CTA synchronisation, 4-5x more SMs busy than one CTA per block.
// 512 threads = 32 (rows tx) x 16 (columns ty); thread owns rows {tx+32a, a<NR} of column ty.
template <int NR>
__global__ void __launch_bounds__(512)
psdscale_small_kernel(const int *ns, const long long *offs, const int *poffs, const double *u, const int *perm,
                      const double *x, int transp, double *y) {
  extern __shared__ double sm[];
  constexpr int NP = 32 * NR, LD = NP + 1;
  const int n = ns[blockIdx.x];
  const int c0 = blockIdx.y * PSD_CS;
  if (c0 >= n) return;
  double *T = sm, *X = sm + NP * LD, *W = X + NP * LD;      // W: NP x PSD_CS (ld = LD)
  const double *U = u + offs[blockIdx.x], *Xg = x + offs[blockIdx.x];
  double *Yg = y + offs[blockIdx.x];
  const int *p = perm ? perm + poffs[blockIdx.x] : nullptr;
  const bool prep = p && !transp, postp = p && transp;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;      // ty < 16
  {  // stage T and X: warp ty takes columns ty, ty+16, ...; lane tx rows tx+32a (no division in the index math)
    int pi[NR];
#pragma unroll
    for (int a = 0; a < NR; a++) pi[a] = (prep && tx + 32 * a < n) ? p[tx + 32 * a] : tx + 32 * a;
    for (int k = ty; k < NP; k += 16) {
      const long long pk = (prep && k < n) ? p[k] : k;
#pragma unroll
      for (int a = 0; a < NR; a++) {
        const int i = tx + 32 * a;
        double tv = 0.0, xv = 0.0;
        if (i < n && k < n) {
          const bool keep = transp ? (i <= k) : (i >= k);        // triu : tril  of the stored array
          tv = keep ? U[i + (long long)k * n] : 0.0;
          xv = Xg[pi[a] + pk * n];
        }
        T[i + k * LD] = tv;
        X[i + k * LD] = xv;
      }
    }
  }
  __syncthreads();
  const int c = c0 + ty;
  {  // W(i,c) = sum_k X(i,k) T(k,c); T(k,c) is zero for k > c (triu) / k < c (tril)
    double acc[NR] = {};
    if (c < n) {
      const int klo = transp ? 0 : c, khi = transp ? c + 1 : n;
#pragma unroll 4
      for (int k = klo; k < khi; k++) {
        const double bv = T[k + c * LD];
#pragma unroll
        for (int a = 0; a < NR; a++) acc[a] += X[tx + 32 * a + k * LD] * bv;
      }
    }
#pragma unroll
    for (int a = 0; a < NR; a++) W[tx + 32 * a + ty * LD] = acc[a];
  }
  __syncthreads();
  {  // Y(i,c) = sum_k T(k,i) W(k,c)
    double acc[NR] = {};
    if (c < n) {
#pragma unroll 4
      for (int k = 0; k < n; k++) {
        const double bv = W[k + ty * LD];
#pragma unroll
        for (int a = 0; a < NR; a++) acc[a] += T[k + (tx + 32 * a) * LD] * bv;
      }
#pragma unroll
      for (int a = 0; a < NR; a++) {
        const int i = tx + 32 * a;
        if (i < n) {
          if (postp) Yg[p[i] + (long long)p[c] * n] = acc[a];
          else Yg[i + (long long)c * n] = acc[a];
        }
      }
    }
  }
}

// Same slab decomposition with the two products on the FP64 tensor pipe (DMMA.8x8x4): X and T stay in their
// natural layouts, padded so that every fragment load is two shared-memory wavefronts (the minimum for doubles):
//   A fragments (row fastest) come from X, ld = NP+8 (2 ld = 16 mod 32 words);
//   fragments that walk k inside a column (B of stage 1: T(k,c); A of stage 2: T(k,i)) come from T, ld = NP+4;
//   W = X T is written transposed (Wt[c][k], ld 24) so that stage 2 reads it as a B operand.
// Warp w owns the 8-row strip w of the result (both 8-column fragments of the 16-column slab); the k-ranges skip the
// structural zeros of the triangular factor.
// The kernel computes a general small congruence Y = T' X T per block, which is also what psdframeit
// (Qb' diag(lab) Qb) and psdinvjmul (Qb Ys Qb', jdiv, Qb' M Qb) are:
//   T  = tsrc or tsrc' (ttrans), optionally masked to its upper (tmask 1) / lower (tmask 2) triangle;
//   X  = xsrc, or xsrc(perm,perm) (prep), or the symmetric matrix held in tril(xsrc) (xsym), or diag(xdiag);
//   Y  : optional jdiv  y_ij *= 2/(l_i+l_j), y_jj /= l_j  (psdinvjmul.c:69-84), then either stored as computed
//        (optionally to (perm,perm), postp) or, symout, the lower triangle is stored and mirrored (exact symmetry).
struct CongArgs {
  const double *tsrc, *xsrc, *xdiag, *jdiv;
  const int *perm;
  int tmask, ttrans, xsym, prep, postp, symout;
};
template <int NR>
__global__ void __launch_bounds__(512)
psdscale_small_dmma_kernel(const int *ns, const long long *offs, const int *poffs, CongArgs A, double *y) {
  extern __shared__ double sm[];
  constexpr int NP = 32 * NR, LDX = NP + 8, LDT = NP + 4, LDW = 24;
  const int n = ns[blockIdx.x];
  const int c0 = blockIdx.y * PSD_CS;
  if (c0 >= n) return;
  double *X = sm, *T = X + NP * LDX, *Wt = T + NP * LDT;          // Wt: [k][c'] as c' + k*LDW
  const double *U = A.tsrc + offs[blockIdx.x];
  const double *Xg = A.xsrc ? A.xsrc + offs[blockIdx.x] : nullptr;
  const double *xd = A.xdiag ? A.xdiag + poffs[blockIdx.x] : nullptr;
  const double *jl = A.jdiv ? A.jdiv + poffs[blockIdx.x] : nullptr;
  double *Yg = y + offs[blockIdx.x];
  const int *p = A.perm ? A.perm + poffs[blockIdx.x] : nullptr;
  const bool prep = p && A.prep, postp = p && A.postp;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  {
    int pi[NR];
#pragma unroll
    for (int a = 0; a < NR; a++) pi[a] = (prep && tx + 32 * a < n) ? p[tx + 32 * a] : tx + 32 * a;
    for (int k = ty; k < NP; k += 16) {
      const long long pk = (prep && k < n) ? p[k] : k;
#pragma unroll
      for (int a = 0; a < NR; a++) {
        const int i = tx + 32 * a;
        double tv = 0.0, xv = 0.0;
        if (i < n && k < n) {
          const bool keep = A.tmask == 0 || (A.tmask == 1 ? (i <= k) : (i >= k));
          tv = keep ? (A.ttrans ? U[k + (long long)i * n] : U[i + (long long)k * n]) : 0.0;
          if (xd) xv = (i == k) ? xd[i] : 0.0;
          else if (A.xsym) xv = Xg[max(i, k) + (long long)min(i, k) * n];
          else xv = Xg[pi[a] + pk * n];
        }
        T[i + k * LDT] = tv;
        X[i + k * LDX] = xv;
      }
    }
  }
  __syncthreads();
  const int warp = ty, qr = tx >> 2, qc = tx & 3;
  const int r8 = warp * 8;                           // this warp's 8-row strip
  const bool active = r8 < n;
  // ---- stage 1: W(i, c0+c') = sum_k X(i,k) T(k, c0+c'),  T(k,c) = 0 for k > c (triu) / k < c (tril)
  if (active) {
    double c00 = 0.0, c01 = 0.0, c10 = 0.0, c11 = 0.0;
    const int klo = A.tmask == 2 ? (c0 & ~3) : 0, khi = A.tmask == 1 ? min(n, c0 + PSD_CS) : n;
    for (int k4 = klo; k4 < khi; k4 += 4) {
      const double af = X[(r8 + qr) + (k4 + qc) * LDX];
      const double b0 = T[(k4 + qc) + (c0 + qr) * LDT], b1 = T[(k4 + qc) + (c0 + 8 + qr) * LDT];
      dmma_m8n8k4(c00, c01, af, b0);
      dmma_m8n8k4(c10, c11, af, b1);
    }
    // C fragment: row qr, columns 2qc, 2qc+1 of each 8-column fragment
    Wt[(2 * qc) + (r8 + qr) * LDW] = c00; Wt[(2 * qc + 1) + (r8 + qr) * LDW] = c01;
    Wt[(8 + 2 * qc) + (r8 + qr) * LDW] = c10; Wt[(8 + 2 * qc + 1) + (r8 + qr) * LDW] = c11;
  }
  __syncthreads();
  // ---- stage 2: Y(i, c0+c') = sum_k T(k,i) W(k,c'),  T(k,i) = 0 for k > i (triu) / k < i (tril)
  if (active && !(A.symout && r8 + 8 <= c0)) {        // symout: strips entirely above the slab's diagonal are mirrored
    double c00 = 0.0, c01 = 0.0, c10 = 0.0, c11 = 0.0;
    const int klo = A.tmask == 2 ? (r8 & ~3) : 0, khi = A.tmask == 1 ? min(n, r8 + 8) : n;
    for (int k4 = klo; k4 < khi; k4 += 4) {
      const double af = T[(k4 + qc) + (r8 + qr) * LDT];                 // A(i,k) = T(k,i)
      const double b0 = Wt[qr + (k4 + qc) * LDW], b1 = Wt[(8 + qr) + (k4 + qc) * LDW];
      dmma_m8n8k4(c00, c01, af, b0);
      dmma_m8n8k4(c10, c11, af, b1);
    }
    const int i = r8 + qr;
    if (i < n) {
      const double v[4] = {c00, c01, c10, c11};
#pragma unroll
      for (int e = 0; e < 4; e++) {
        const int c = c0 + (e >> 1) * 8 + 2 * qc + (e & 1);
        if (c < n) {
          double val = v[e];
          if (jl) val = (i == c) ? val / jl[c] : val * (2.0 / (jl[i] + jl[c]));
          if (A.symout) {
            if (i >= c) { Yg[i + (long long)c * n] = val; if (i != c) Yg[c + (long long)i * n] = val; }
          } else if (postp) Yg[p[i] + (long long)p[c] * n] = val;
          else Yg[i + (long long)c * n] = val;
        }
      }
    }
  }
}

// ---------------------------------------------------------------- Hermitian PSD blocks
// A Hermitian block of order n arrives as [vec Re; vec Im] (2 n^2 doubles).  The complex algebra runs on
// the real embedding E(Z) = [[Re Z, -Im Z],[Im Z, Re Z]] (a *-homomorphism: E(Z^H) = E(Z)', E(XY) = E(X)E(Y)),
// i.e. as a real block of order 2n through the same DMMA products; real blocks are carried along as they are.
struct HermBlk { int n, cplx, poff, pad; long long raw_off, emb_off; };

// emb = E(op(raw)):  op = gather by perm (src(P[p],P[q])), triangular mask on the source (1: keep row<=col,
// 2: keep row>=col), conjugate transpose (tc).
__global__ void herm_embed_kernel(const HermBlk *blks, const double *raw, double *emb, const int *perm, int tc, int mask) {
  const HermBlk B = blks[blockIdx.y];
  const int n = B.n, ne = B.cplx ? 2 * n : n;
  const double *re = raw + B.raw_off, *im = re + (long long)n * n;
  double *E = emb + B.emb_off;
  const int *P = perm ? perm + B.poff : nullptr;
  const long long tot = (long long)n * n;
  for (long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x; idx < tot; idx += (long long)gridDim.x * blockDim.x) {
    const int p = (int)(idx % n), q = (int)(idx / n);
    int sp = tc ? q : p, sq = tc ? p : q;
    if (P) { sp = P[sp]; sq = P[sq]; }
    bool keep = mask == 0 || mask == 3 || (mask == 1 ? sp <= sq : sp >= sq);
    bool flip = false;                                     // mask 3: Hermitian completion from the lower triangle
    if (mask == 3 && sp < sq) { const int t = sp; sp = sq; sq = t; flip = true; }
    const long long si = sp + (long long)sq * n;
    double zr = keep ? re[si] : 0.0, zi = (keep && B.cplx) ? im[si] : 0.0;
    if (tc != flip) zi = -zi;
    if (mask == 3 && sp == sq) zi = 0.0;
    E[p + (long long)q * ne] = zr;
    if (B.cplx) {
      E[(p + n) + (long long)(q + n) * ne] = zr;
      E[(p + n) + (long long)q * ne] = zi;
      E[p + (long long)(q + n) * ne] = -zi;
    }
  }
}
// raw(P[p],P[q]) (or raw(p,q)) = the complex entry (p,q) of emb; the imaginary diagonal can be forced to 0.
__global__ void herm_extract_kernel(const HermBlk *blks, const double *emb, double *raw, const int *perm, int zero_imag_diag) {
  const HermBlk B = blks[blockIdx.y];
  const int n = B.n, ne = B.cplx ? 2 * n : n;
  double *re = raw + B.raw_off, *im = re + (long long)n * n;
  const double *E = emb + B.emb_off;
  const int *P = perm ? perm + B.poff : nullptr;
  const long long tot = (long long)n * n;
  for (long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x; idx < tot; idx += (long long)gridDim.x * blockDim.x) {
    const int p = (int)(idx % n), q = (int)(idx / n);
    const int dp = P ? P[p] : p, dq = P ? P[q] : q;
    const long long di = dp + (long long)dq * n;
    re[di] = E[p + (long long)q * ne];
    if (B.cplx) im[di] = (zero_imag_diag && dp == dq) ? 0.0 : E[(p + n) + (long long)q * ne];
  }
}

// Columns of Qb = H_0 ... H_{n-2} diag(qsgn) for a Hermitian block, H_c = I - c_c c_c^H / beta_c (reflect.c:218-262:
// frames [Re c | Im c | beta], the last column of c is the complex sign vector).  One warp per column, written
// straight into the real embedding: column j of E(Qb) = [Re q; Im q], column j+n = [-Im q; Re q].
__global__ void __launch_bounds__(256)
householder_q_cplx_kernel(const HermBlk *blks, const int *grp_blk, const int *grp_j0, const long long *fr_off,
                          const double *frms, double *Qe) {
  const int k = grp_blk[blockIdx.x];
  const HermBlk B = blks[k];
  const int n = B.n, ne = 2 * n;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int j = grp_j0[blockIdx.x] + warp;
  if (j >= n) return;
  const double *cr = frms + fr_off[k], *ci = cr + (long long)n * n, *beta = ci + (long long)n * n;
  double *qr = Qe + B.emb_off + (long long)j * ne, *qi = qr + n;
  const double sr = cr[(long long)(n - 1) * n + j], si = ci[(long long)(n - 1) * n + j];
  for (int i = lane; i < n; i += 32) { qr[i] = (i == j) ? sr : 0.0; qi[i] = (i == j) ? si : 0.0; }
  __syncwarp();
  for (int c = min(j, n - 2); c >= 0; c--) {
    const double *vr = cr + (long long)c * n, *vi = ci + (long long)c * n;
    double tr = 0.0, ti = 0.0;                           // t = v^H q
    for (int i = c + lane; i < n; i += 32) {
      tr += vr[i] * qr[i] + vi[i] * qi[i];
      ti += vr[i] * qi[i] - vi[i] * qr[i];
    }
    for (int o = 16; o > 0; o >>= 1) { tr += __shfl_xor_sync(0xffffffffu, tr, o); ti += __shfl_xor_sync(0xffffffffu, ti, o); }
    const double ar = -tr / beta[c], ai = -ti / beta[c];
    for (int i = c + lane; i < n; i += 32) {
      const double xr = vr[i], xi = vi[i];
      qr[i] += ar * xr - ai * xi;
      qi[i] += ar * xi + ai * xr;
    }
    __syncwarp();
  }
  double *q2 = Qe + B.emb_off + (long long)(j + n) * ne;
  for (int i = lane; i < n; i += 32) { q2[i] = -qi[i]; q2[n + i] = qr[i]; }
}

// Real frames of the mixed layout -> the embedded layout; Hermitian slots get "no reflection" frames (zero
// vectors, beta = 1) so that the real builder leaves an identity there (it is overwritten afterwards).
__global__ void herm_frames_kernel(const HermBlk *blks, const long long *fr_off, const double *frms, double *Femb) {
  const HermBlk B = blks[blockIdx.y];
  const int n = B.n, ne = B.cplx ? 2 * n : n;
  const double *F = frms + fr_off[blockIdx.y];
  double *E = Femb + B.emb_off;
  const long long tot = (long long)ne * ne;
  for (long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x; idx < tot; idx += (long long)gridDim.x * blockDim.x) {
    if (!B.cplx) E[idx] = F[idx];
    else E[idx] = (idx / ne == ne - 1) ? 1.0 : 0.0;
  }
}

static std::map<Hash128, sb200_psd_plan *> g_psd_plans;

}  // namespace sb

using namespace sb;

static int psd_build(sb200_psd_plan *pl, sb_idx nblk, const sb_idx *n) {
  pl->nblk = (int)nblk;
  long long off = 0; int po = 0;
  for (sb_idx k = 0; k < nblk; k++) {
    SB_CHECK(n[k] >= 1 && n[k] < 46340, "PSD block order %lld out of range", (long long)n[k]);
    pl->n.push_back((int)n[k]); pl->off.push_back(off); pl->poff.push_back(po);
    off += n[k] * n[k]; po += (int)n[k];
    pl->maxn = std::max(pl->maxn, (int)n[k]);
  }
  pl->lenud = off; pl->sumn = po;
  std::vector<GemmDesc> ichol, s1lo, s1up, s2lo, s2up, dfull, dlower;
  std::vector<int> qblk, qj0;
  std::vector<GemmTile> tfull, tlower;
  for (int k = 0; k < pl->nblk; k++) {
    int nk = pl->n[k]; long long o = pl->off[k];
    GemmDesc g{};
    g.gatherOff = -1; g.lda = g.ldb = g.ldc = nk; g.M = g.N = g.K = nk; g.alpha = 1.0; g.accumulate = 0;
    g.offA = g.offB = g.offC = o;
    // invcholfac: A = B = Tt (k <= row), lower only
    GemmDesc a = g; a.a_tri = TRI_K_LE_ROW; a.b_tri = TRI_K_LE_ROW; a.lower = 1; ichol.push_back(a);
    // psdscale stage 1: Wt = Tt * X'   (A = Tt, B = X)
    GemmDesc b = g; b.lower = 0; b.b_tri = TRI_NONE;
    b.a_tri = TRI_K_GE_ROW; s1lo.push_back(b);          // T = tril(U): Tt(c,k) nonzero for k >= c
    b.a_tri = TRI_K_LE_ROW; s1up.push_back(b);          // T = triu(U)
    // stage 2: Y = Tt * Wt'
    b.a_tri = TRI_K_GE_ROW; s2lo.push_back(b);
    b.a_tri = TRI_K_LE_ROW; s2up.push_back(b);
    GemmDesc f = g; f.a_tri = f.b_tri = TRI_NONE; f.lower = 0; dfull.push_back(f);
    f.lower = 1; dlower.push_back(f);
    for (int j0 = 0; j0 < nk; j0 += 8) { qblk.push_back(k); qj0.push_back(j0); }
    gemm_add_tiles(tfull, k, nk, nk, false);
    gemm_add_tiles(tlower, k, nk, nk, true);
  }
  pl->ntiles_full = (int)tfull.size(); pl->ntiles_lower = (int)tlower.size();
  // ---- compact-WY schedule
  {
    const int nld = (pl->maxn + 1) & ~1;
    pl->wy_rows_smem = sizeof(double) * ((size_t)WY_RW * nld + 2 * WY_CH * (WYB + 1) + 2 * WY_RW * WYB + WYB * (WYB + 1));
    // small blocks: the one-warp-per-column kernel is a single short launch (the row kernel needs the T factors
    // first: two launches)
    pl->wy_rows = pl->maxn > 96 && pl->wy_rows_smem <= 220 * 1024;
    if (const char *e = getenv("SB200_WY_GEMM_MIN_N")) if (pl->maxn >= atoi(e)) pl->wy_rows = false;     // tests: force the GEMM path
    pl->wy = pl->maxn > 96 && !pl->wy_rows;
  }
  if (pl->wy || pl->wy_rows) {
    const int wyb = pl->wy ? WYBIG : WYB;          // the GEMM path uses wide panels: its products need N, K >> 32 to be efficient
    pl->wyb = wyb;
    std::vector<GemmDesc> wd;
    std::vector<GemmTile> wt;
    std::vector<int> pblk, pidx;
    std::vector<long long> toff(pl->nblk, 0), yoff(pl->nblk, 0);
    long long tcount = 0, ycount = 0;
    int maxP = 0;
    for (int k = 0; k < pl->nblk; k++) {
      const int nk = pl->n[k], P = (nk - 1 + wyb - 1) / wyb;
      toff[k] = tcount; yoff[k] = ycount;
      for (int p2 = 0; p2 < P; p2++) { pblk.push_back(k); pidx.push_back(p2); }
      tcount += P; ycount += (long long)nk * wyb;
      maxP = std::max(maxP, P);
    }
    pl->wy_npanels = (int)pblk.size(); pl->wy_steps = maxP;
    for (int st = 0; st < maxP; st++) {
      sb200_psd_plan::WyStep W{};
      std::vector<GemmDesc> g1, g2, g3;
      std::vector<GemmTile> t1, t2, t3;
      for (int k = 0; k < pl->nblk; k++) {
        const int nk = pl->n[k], P = (nk - 1 + wyb - 1) / wyb;
        const int p2 = P - 1 - st;
        if (p2 < 0) continue;
        const int c0 = p2 * wyb, bp = std::min(wyb, nk - 1 - c0), np = nk - c0;
        const long long sub = pl->off[k] + c0 + (long long)c0 * nk;      // (c0, c0) corner inside the block
        GemmDesc a{}; a.gatherOff = -1; a.alpha = 1.0;
        // Y(i,c) = sum_r R(i,r) V(r,c):  A = R sub-block, B = F' rows c (k >= row mask)
        a.offA = sub; a.lda = nk; a.a_tri = TRI_NONE;
        a.offB = sub; a.ldb = nk; a.b_tri = TRI_K_GE_ROW;
        a.offC = yoff[k]; a.ldc = nk; a.M = np; a.N = bp; a.K = np; a.lower = 0; a.accumulate = 0;
        gemm_add_tiles(t1, (int)g1.size(), np, bp, false); g1.push_back(a);
        // Y2 = Y T'
        GemmDesc b{}; b.gatherOff = -1; b.alpha = 1.0;
        b.offA = yoff[k]; b.lda = nk; b.a_tri = TRI_NONE;
        b.offB = (toff[k] + p2) * (long long)wyb * wyb; b.ldb = wyb; b.b_tri = TRI_NONE;
        b.offC = yoff[k]; b.ldc = nk; b.M = np; b.N = bp; b.K = bp; b.lower = 0; b.accumulate = 0;
        gemm_add_tiles(t2, (int)g2.size(), np, bp, false); g2.push_back(b);
        // R(i,r) -= sum_c Y2(i,c) V(r,c):  B = F rows r (k <= row mask)
        GemmDesc c{}; c.gatherOff = -1; c.alpha = -1.0;
        c.offA = yoff[k]; c.lda = nk; c.a_tri = TRI_NONE;
        c.offB = sub; c.ldb = nk; c.b_tri = TRI_K_LE_ROW;
        c.offC = sub; c.ldc = nk; c.M = np; c.N = np; c.K = bp; c.lower = 0; c.accumulate = 1;
        gemm_add_tiles(t3, (int)g3.size(), np, np, false); g3.push_back(c);
      }
      auto push = [&](std::vector<GemmDesc> &g, std::vector<GemmTile> &t, int &d0, int &tt0, int &nt) {
        d0 = (int)wd.size(); tt0 = (int)wt.size(); nt = (int)t.size();
        for (auto &x : t) x.prob += d0;
        wd.insert(wd.end(), g.begin(), g.end()); wt.insert(wt.end(), t.begin(), t.end());
      };
      push(g1, t1, W.d1, W.t1, W.n1); push(g2, t2, W.d2, W.t2, W.n2); push(g3, t3, W.d3, W.t3, W.n3);
      pl->wy_sched.push_back(W);
    }
    if (pl->wy) {                                    // G_p = V_p' V_p for every panel of every block, one launch
      std::vector<GemmDesc> gg; std::vector<GemmTile> gt;
      for (int k = 0; k < pl->nblk; k++) {
        const int nk = pl->n[k], P = (nk - 1 + wyb - 1) / wyb;
        for (int p2 = 0; p2 < P; p2++) {
          const int c0 = p2 * wyb, bp = std::min(wyb, nk - 1 - c0), np = nk - c0;
          const long long sub = pl->off[k] + c0 + (long long)c0 * nk;
          GemmDesc g{}; g.gatherOff = -1; g.alpha = 1.0;
          g.offA = sub; g.lda = nk; g.a_tri = TRI_K_GE_ROW;          // F' rows = reflectors, k = matrix row >= reflector index
          g.offB = sub; g.ldb = nk; g.b_tri = TRI_K_GE_ROW;
          g.offC = (toff[k] + p2) * (long long)wyb * wyb; g.ldc = wyb; g.M = bp; g.N = bp; g.K = np; g.lower = 0; g.accumulate = 0;
          gemm_add_tiles(gt, (int)gg.size(), bp, bp, false); gg.push_back(g);
        }
      }
      pl->wy_gd = (int)wd.size(); pl->wy_gt = (int)wt.size(); pl->wy_gn = (int)gt.size();
      for (auto &x : gt) x.prob += pl->wy_gd;
      wd.insert(wd.end(), gg.begin(), gg.end()); wt.insert(wt.end(), gt.begin(), gt.end());
      SB_TRY(pl->d_wy_G.alloc((size_t)tcount * wyb * wyb));
    }
    SB_TRY(pl->d_wy_desc.upload(wd)); SB_TRY(pl->d_wy_tiles.upload(wt));
    SB_TRY(pl->d_wy_pblk.upload(pblk)); SB_TRY(pl->d_wy_pidx.upload(pidx)); SB_TRY(pl->d_wy_toff.upload(toff));
    SB_TRY(pl->d_wy_T.alloc((size_t)tcount * wyb * wyb));
    SB_TRY(pl->d_wy_Y.alloc((size_t)ycount)); SB_TRY(pl->d_wy_Y2.alloc((size_t)ycount));
  }
  SB_TRY(pl->d_n.upload(pl->n)); SB_TRY(pl->d_off.upload(pl->off)); SB_TRY(pl->d_poff.upload(pl->poff));
  SB_TRY(pl->d_desc_ichol.upload(ichol));
  SB_TRY(pl->d_desc_s1_lo.upload(s1lo)); SB_TRY(pl->d_desc_s1_up.upload(s1up));
  SB_TRY(pl->d_desc_s2_lo.upload(s2lo)); SB_TRY(pl->d_desc_s2_up.upload(s2up));
  SB_TRY(pl->d_desc_full.upload(dfull)); SB_TRY(pl->d_desc_lower.upload(dlower));
  pl->nqgroups = (int)qblk.size();
  SB_TRY(pl->d_qcol_blk.upload(qblk)); SB_TRY(pl->d_qcol_j0.upload(qj0));
  SB_TRY(pl->d_tiles_full.upload(tfull)); SB_TRY(pl->d_tiles_lower.upload(tlower));
  SB_TRY(pl->d_Tt.alloc((size_t)pl->lenud)); SB_TRY(pl->d_Wt.alloc((size_t)pl->lenud));
  SB_TRY(pl->d_Xp.alloc((size_t)pl->lenud)); SB_TRY(pl->d_Y.alloc((size_t)pl->lenud));
  SB_TRY(pl->d_perm.alloc((size_t)std::max<long long>(pl->sumn, 1)));
  SB_CUDA(cudaStreamSynchronize(ctx().stream));
  return 0;
}

extern "C" {

int sb200_psd_plan_get(sb200_psd_plan **plan, sb_idx nblk, const sb_idx *n) {
  SB_TRY(ensure_init());
  Hash128 key = fnv1a(n, sizeof(sb_idx) * nblk, fnv1a(&nblk, sizeof nblk));
  auto it = g_psd_plans.find(key);
  if (it != g_psd_plans.end()) { *plan = it->second; return 0; }
  sb200_psd_plan *pl = new sb200_psd_plan();
  int rc = psd_build(pl, nblk, n);
  if (rc) { delete pl; return rc; }
  g_psd_plans[key] = pl;
  *plan = pl;
  return 0;
}
sb_idx sb200_psd_plan_lenud(const sb200_psd_plan *pl) { return pl->lenud; }
// device-side block table (orders, offsets in a lenud vector) for kernels of other translation units
int sb200_psd_plan_blocks(sb200_psd_plan *pl, const int **n_dev, const long long **off_dev, int *nblk, int *maxn) {
  *n_dev = pl->d_n.p; *off_dev = pl->d_off.p; *nblk = pl->nblk; *maxn = pl->maxn;
  return 0;
}
sb_idx sb200_psd_plan_sumn(const sb200_psd_plan *pl) { return pl->sumn; }

static dim3 blk_grid(const sb200_psd_plan *pl, int per) {
  long long t = (long long)pl->maxn * pl->maxn;
  int gx = (int)std::min<long long>((t + per - 1) / per, 1024);
  return dim3(std::max(gx, 1), pl->nblk);
}

// Y = T' X T for every block of a plan whose blocks are at most PSD_SMALL_MAX wide (one fused DMMA kernel).
static int small_congruence(sb200_psd_plan *pl, const CongArgs &A, double *y_dev) {
  const int NR = (pl->maxn + 31) / 32, NP = 32 * NR;
  const size_t shm = sizeof(double) * ((size_t)NP * (NP + 8) + (size_t)NP * (NP + 4) + (size_t)NP * 24);
  const dim3 grid(pl->nblk, (pl->maxn + PSD_CS - 1) / PSD_CS);
  cudaStream_t st = ctx().stream;
  auto launch = [&](auto kern) -> int {
    if (shm > 48 * 1024) SB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)shm));
    kern<<<grid, 512, shm, st>>>(pl->d_n.p, pl->d_off.p, pl->d_poff.p, A, y_dev);
    return 0;
  };
  if (NR == 1) return launch(psdscale_small_dmma_kernel<1>);
  if (NR == 2) return launch(psdscale_small_dmma_kernel<2>);
  return launch(psdscale_small_dmma_kernel<3>);
}

// block-wise symmetric permutation (no symmetric read): column kernel for moderate orders, element kernel otherwise
static int launch_perm(sb200_psd_plan *pl, const int *perm_dev, const double *in, double *out, int gather, cudaStream_t st) {
  if (perm_dev && pl->maxn <= PERM_COLS_MAXN) {
    const size_t shm = sizeof(double) * (size_t)PERM_COLS_W * pl->maxn + sizeof(int) * (size_t)pl->maxn;
    perm_cols_kernel<<<dim3((pl->maxn + PERM_COLS_W - 1) / PERM_COLS_W, pl->nblk), 32 * PERM_COLS_W, shm, st>>>(
        pl->d_n.p, pl->d_off.p, pl->d_poff.p, perm_dev, in, out, gather);
    SB_LAUNCH_CHECK_N("perm_cols_kernel");
    return 0;
  }
  perm_block_kernel<<<blk_grid(pl, 256), 256, 0, st>>>(pl->d_n.p, pl->d_off.p, pl->d_poff.p, perm_dev, in, out, gather, 0);
  SB_LAUNCH_CHECK_N("perm_block_kernel");
  return 0;
}

// y = invcholfac(u, K, perm): perm_dev is int32 0-based (length sum n_k) or NULL.
int sb200_invcholfac_dev(sb200_psd_plan *pl, const double *u_dev, const int *perm_dev, double *y_dev) {
  SB_TRY(ensure_init());
  if (pl->nblk == 0) return 0;
  cudaStream_t st = ctx().stream;
  tri_transpose_kernel<<<dim3(std::min(1024, ((pl->maxn + 31) / 32) * ((pl->maxn + 31) / 32)), pl->nblk), dim3(32, 8), 0, st>>>(
      pl->d_n.p, pl->d_off.p, u_dev, pl->d_Tt.p, 1);
  SB_LAUNCH_CHECK_N("tri_transpose_kernel");
  gemm_nt_launch(pl->ntiles_lower, ctx().sm_count, st, pl->d_desc_ichol.p, pl->d_tiles_lower.p, pl->d_Tt.p, pl->d_Tt.p,
                                                   pl->d_Wt.p, nullptr);
  SB_LAUNCH_CHECK_N("gemm_nt_kernel");
  perm_block_kernel<<<blk_grid(pl, 256), 256, 0, st>>>(pl->d_n.p, pl->d_off.p, pl->d_poff.p, perm_dev, pl->d_Wt.p, y_dev, 0, 1);
  SB_LAUNCH_CHECK_N("perm_block_kernel");
  return 0;
}

// y = psdscale(ud, x, K, transp): x_dev/y_dev are the PSD parts (lenud).  perm_dev as above
// (NULL when ud.perm is empty or ud is a plain vector).
int sb200_psdscale_dev(sb200_psd_plan *pl, const double *u_dev, const int *perm_dev, const double *x_dev,
                       int transp, double *y_dev) {
  SB_TRY(ensure_init());
  if (pl->nblk == 0) return 0;
  cudaStream_t st = ctx().stream;
  if (pl->maxn <= PSD_SMALL_MAX) {
    const int NR = (pl->maxn + 31) / 32, NP = 32 * NR;
    static const bool use_fma = getenv("SB200_PSDSCALE_FMA") != nullptr;       // the first (FP64 FMA) version, for comparison
    const size_t shm = use_fma ? sizeof(double) * (2 * (size_t)NP + PSD_CS) * (NP + 1)
                               : sizeof(double) * ((size_t)NP * (NP + 8) + (size_t)NP * (NP + 4) + (size_t)NP * 24);
    auto launch = [&](auto kern) -> int {
      if (shm > 48 * 1024) SB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)shm));
      kern<<<dim3(pl->nblk, (pl->maxn + PSD_CS - 1) / PSD_CS), 512, shm, st>>>(pl->d_n.p, pl->d_off.p, pl->d_poff.p, u_dev, perm_dev, x_dev, transp, y_dev);
      return 0;
    };
    (void)NP;
    if (use_fma) {
      if (NR == 1) SB_TRY(launch(psdscale_small_kernel<1>));
      else if (NR == 2) SB_TRY(launch(psdscale_small_kernel<2>));
      else SB_TRY(launch(psdscale_small_kernel<3>));
    } else {
      CongArgs A{u_dev, x_dev, nullptr, nullptr, perm_dev, transp ? 1 : 2, 0, 0, transp ? 0 : 1, transp ? 1 : 0, 0};
      SB_TRY(small_congruence(pl, A, y_dev));
    }
    SB_LAUNCH_CHECK_N("psdscale_small_kernel");
    return 0;
  }
  tri_transpose_kernel<<<dim3(std::min(1024, ((pl->maxn + 31) / 32) * ((pl->maxn + 31) / 32)), pl->nblk), dim3(32, 8), 0, st>>>(
      pl->d_n.p, pl->d_off.p, u_dev, pl->d_Tt.p, transp ? 1 : 0);
  SB_LAUNCH_CHECK_N("tri_transpose_kernel");
  const double *xs = x_dev;
  if (perm_dev && !transp) {          // prep: X(perm,perm)   (psdscale.m:94-99)
    SB_TRY(launch_perm(pl, perm_dev, x_dev, pl->d_Xp.p, 1, st));
    xs = pl->d_Xp.p;
  }
  gemm_nt_launch(pl->ntiles_full, ctx().sm_count, st, (transp ? pl->d_desc_s1_up : pl->d_desc_s1_lo).p, pl->d_tiles_full.p,
                                                  pl->d_Tt.p, xs, pl->d_Wt.p, nullptr);
  SB_LAUNCH_CHECK_N("gemm_nt_kernel");
  bool postp = perm_dev && transp;
  gemm_nt_launch(pl->ntiles_full, ctx().sm_count, st, (transp ? pl->d_desc_s2_up : pl->d_desc_s2_lo).p, pl->d_tiles_full.p,
                                                  pl->d_Tt.p, pl->d_Wt.p, postp ? pl->d_Y.p : y_dev, nullptr);
  SB_LAUNCH_CHECK_N("gemm_nt_kernel");
  if (postp) {                         // XX(PP,PP) = XX   (psdscale.m:104-109)
    SB_TRY(launch_perm(pl, perm_dev, pl->d_Y.p, y_dev, 0, st));
  }
  return 0;
}

static int upload_perm(sb200_psd_plan *pl, const sb_idx *perm, const int **out) {
  *out = nullptr;
  if (!perm) return 0;
  std::vector<int> p32((size_t)pl->sumn);
  for (int k = 0; k < pl->nblk; k++)
    for (int i = 0; i < pl->n[k]; i++) {
      sb_idx v = perm[pl->poff[k] + i];
      SB_CHECK(v >= 0 && v < pl->n[k], "perm entry out of range in PSD block %d", k);
      p32[pl->poff[k] + i] = (int)v;
    }
  SB_CUDA(cudaMemcpyAsync(pl->d_perm.p, p32.data(), sizeof(int) * p32.size(), cudaMemcpyHostToDevice, ctx().stream));
  SB_CUDA(cudaStreamSynchronize(ctx().stream));
  *out = pl->d_perm.p;
  return 0;
}

// Host entries.  perm: 0-based within each block (NULL = none).
int sb200_invcholfac(sb_idx nblk, const sb_idx *n, const double *u, const sb_idx *perm, double *y) {
  sb200_psd_plan *pl = nullptr;
  SB_TRY(sb200_psd_plan_get(&pl, nblk, n));
  if (pl->lenud == 0) return 0;
  arena_reset();
  // d.u is the same array for invcholfac, the psdscale calls and urotorder of one IPM iteration: its device copy is
  // found again by content (mirror_input), only the first of those calls pays the upload
  const double *du = (const double *)mirror_input(u, sizeof(double) * pl->lenud);
  double *dy = arena<double>((size_t)pl->lenud);
  SB_CHECK(du && dy, "invcholfac: out of device memory");
  const int *dperm;
  SB_TRY(upload_perm(pl, perm, &dperm));
  SB_TRY(sb200_invcholfac_dev(pl, du, dperm, dy));
  SB_CUDA(cudaMemcpyAsync(y, dy, sizeof(double) * pl->lenud, cudaMemcpyDeviceToHost, ctx().stream));
  SB_CUDA(cudaStreamSynchronize(ctx().stream));
  return 0;
}

int sb200_psdscale(sb_idx nblk, const sb_idx *n, const double *u, const sb_idx *perm, const double *x, int transp, double *y) {
  sb200_psd_plan *pl = nullptr;
  SB_TRY(sb200_psd_plan_get(&pl, nblk, n));
  if (pl->lenud == 0) return 0;
  arena_reset();
  const double *du = (const double *)mirror_input(u, sizeof(double) * pl->lenud);
  double *dx = arena<double>((size_t)pl->lenud), *dy = arena<double>((size_t)pl->lenud);
  SB_CHECK(du && dx && dy, "psdscale: out of device memory");
  const int *dperm;
  SB_TRY(upload_perm(pl, perm, &dperm));
  SB_CUDA(cudaMemcpyAsync(dx, x, sizeof(double) * pl->lenud, cudaMemcpyHostToDevice, ctx().stream));
  SB_TRY(sb200_psdscale_dev(pl, du, dperm, dx, transp, dy));
  SB_CUDA(cudaMemcpyAsync(y, dy, sizeof(double) * pl->lenud, cudaMemcpyDeviceToHost, ctx().stream));
  SB_CUDA(cudaStreamSynchronize(ctx().stream));
  return 0;
}

// ---- Householder-frame operations.  frms_dev: lenud doubles (real blocks); lab/xlab: sum(n_k) doubles.
static int build_q(sb200_psd_plan *pl, const double *frms_dev, bool need_transpose = true) {   // Q -> d_Tt, Q' -> d_Wt
  cudaStream_t st = ctx().stream;
  int tp = (pl->maxn + 31) / 32;
  if (pl->wy_rows) {
    wy_t_kernel<<<pl->wy_npanels, 256, 0, st>>>(pl->d_wy_pblk.p, pl->d_wy_pidx.p, pl->d_n.p, pl->d_off.p, pl->d_wy_toff.p, frms_dev, pl->d_wy_T.p);
    SB_LAUNCH_CHECK_N("wy_t_kernel");
    static bool attr_done = false;
    if (!attr_done) { SB_CUDA(cudaFuncSetAttribute(wy_rows_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 225 * 1024)); attr_done = true; }
    wy_rows_kernel<<<pl->nqgroups, 256, pl->wy_rows_smem, st>>>(pl->d_qcol_blk.p, pl->d_qcol_j0.p, pl->d_n.p, pl->d_off.p, pl->d_wy_toff.p,
                                                                frms_dev, pl->d_wy_T.p, pl->d_Tt.p);
    SB_LAUNCH_CHECK_N("wy_rows_kernel");
    transpose_scale_kernel<<<dim3(std::min(1024, tp * tp), pl->nblk), dim3(32, 8), 0, st>>>(pl->d_n.p, pl->d_off.p, pl->d_poff.p, pl->d_Tt.p, nullptr, pl->d_Wt.p);
    SB_LAUNCH_CHECK_N("transpose_scale_kernel");
    return 0;
  }
  if (pl->wy) {
    // R = Q' accumulated right to left, panel by panel:  R <- R (I - V_p T_p V_p')' = R - (R V_p) T_p' V_p'
    // with panels of 128 reflectors, so that every product of the loop has N or K = 128 (32-wide panels make the
    // rank-32 updates the bulk of the GEMM-engine time of a large block)
    transpose_scale_kernel<<<dim3(std::min(1024, tp * tp), pl->nblk), dim3(32, 8), 0, st>>>(pl->d_n.p, pl->d_off.p, pl->d_poff.p, frms_dev, nullptr, pl->d_Xp.p);   // F'
    SB_LAUNCH_CHECK_N("transpose_scale_kernel");
    gemm_nt_launch(pl->wy_gn, ctx().sm_count, st, pl->d_wy_desc.p, pl->d_wy_tiles.p + pl->wy_gt, pl->d_Xp.p, pl->d_Xp.p, pl->d_wy_G.p, nullptr);
    SB_LAUNCH_CHECK_N("gemm_nt_kernel");
    {
      const size_t shm = sizeof(double) * WYBIG * (WYBIG + 1);
      static bool attr_done = false;
      if (!attr_done) { SB_CUDA(cudaFuncSetAttribute(wy_tinv_big_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)shm)); attr_done = true; }
      wy_tinv_big_kernel<<<pl->wy_npanels, WYBIG, shm, st>>>(pl->d_wy_pblk.p, pl->d_wy_pidx.p, pl->d_n.p, pl->d_off.p, pl->d_wy_toff.p, frms_dev,
                                                           pl->d_wy_G.p, pl->d_wy_T.p);
      SB_LAUNCH_CHECK_N("wy_tinv_big_kernel");
    }
    set_identity_kernel<<<dim3((unsigned)std::min<long long>(((long long)pl->maxn * pl->maxn + 255) / 256, 1024), pl->nblk), 256, 0, st>>>(pl->d_n.p, pl->d_off.p, pl->d_Wt.p);
    SB_LAUNCH_CHECK_N("set_identity_kernel");
    for (auto &W : pl->wy_sched) {
      // descriptors carry absolute indices into d_wy_desc; tiles reference them
      gemm_nt_launch(W.n1, ctx().sm_count, st, pl->d_wy_desc.p, pl->d_wy_tiles.p + W.t1, pl->d_Wt.p, pl->d_Xp.p, pl->d_wy_Y.p, nullptr);
      SB_LAUNCH_CHECK_N("gemm_nt_kernel");
      gemm_nt_launch(W.n2, ctx().sm_count, st, pl->d_wy_desc.p, pl->d_wy_tiles.p + W.t2, pl->d_wy_Y.p, pl->d_wy_T.p, pl->d_wy_Y2.p, nullptr);
      SB_LAUNCH_CHECK_N("gemm_nt_kernel");
      gemm_nt_launch(W.n3, ctx().sm_count, st, pl->d_wy_desc.p, pl->d_wy_tiles.p + W.t3, pl->d_wy_Y2.p, frms_dev, pl->d_Wt.p, nullptr);
      SB_LAUNCH_CHECK_N("gemm_nt_kernel");
    }
    transpose_scale_kernel<<<dim3(std::min(1024, tp * tp), pl->nblk), dim3(32, 8), 0, st>>>(pl->d_n.p, pl->d_off.p, pl->d_poff.p, pl->d_Wt.p, nullptr, pl->d_Tt.p);
    SB_LAUNCH_CHECK_N("transpose_scale_kernel");
    return 0;
  }
  householder_q_kernel<<<pl->nqgroups, 256, 0, st>>>(pl->d_qcol_blk.p, pl->d_qcol_j0.p, pl->d_n.p, pl->d_off.p, frms_dev, pl->d_Tt.p);
  SB_LAUNCH_CHECK_N("householder_q_kernel");
  if (!need_transpose) return 0;
  transpose_scale_kernel<<<dim3(std::min(1024, tp * tp), pl->nblk), dim3(32, 8), 0, st>>>(pl->d_n.p, pl->d_off.p, pl->d_poff.p, pl->d_Tt.p, nullptr, pl->d_Wt.p);
  SB_LAUNCH_CHECK_N("transpose_scale_kernel");
  return 0;
}

// x = psdframeit(lab, frms, K):  X_k = Qb' diag(lab_k) Qb   (psdframeit.c:65-99)
static int psdframeit_core(sb200_psd_plan *pl, const double *lab_dev, double *x_dev);
int sb200_psdframeit_dev(sb200_psd_plan *pl, const double *lab_dev, const double *frms_dev, double *x_dev) {
  SB_TRY(ensure_init());
  if (pl->nblk == 0) return 0;
  if (pl->maxn <= PSD_SMALL_MAX && !pl->wy && !pl->wy_rows) {
    // small blocks: Q by the per-column kernel, then ONE fused congruence  X = Q' diag(lab) Q  (lower triangle mirrored)
    SB_TRY(build_q(pl, frms_dev, false));
    CongArgs A{pl->d_Tt.p, nullptr, lab_dev, nullptr, nullptr, 0, 0, 0, 0, 0, 1};
    SB_TRY(small_congruence(pl, A, x_dev));
    SB_LAUNCH_CHECK_N("small_congruence_kernel");
    return 0;
  }
  SB_TRY(build_q(pl, frms_dev));
  return psdframeit_core(pl, lab_dev, x_dev);
}
// X = Q' diag(lab) Q with Q in d_Tt and Q' in d_Wt
static int psdframeit_core(sb200_psd_plan *pl, const double *lab_dev, double *x_dev) {
  cudaStream_t st = ctx().stream;
  int tp = (pl->maxn + 31) / 32;
  // B(c,k) = lab_k * Qb(k,c): transpose of Q with the k-index scaled -> d_Xp
  transpose_scale_kernel<<<dim3(std::min(1024, tp * tp), pl->nblk), dim3(32, 8), 0, st>>>(pl->d_n.p, pl->d_off.p, pl->d_poff.p, pl->d_Tt.p, lab_dev, pl->d_Xp.p);
  SB_LAUNCH_CHECK_N("transpose_scale_kernel");
  gemm_nt_launch(pl->ntiles_lower, ctx().sm_count, st, pl->d_desc_lower.p, pl->d_tiles_lower.p, pl->d_Wt.p, pl->d_Xp.p, x_dev, nullptr);
  SB_LAUNCH_CHECK_N("gemm_nt_kernel");
  sym_ops_kernel<<<blk_grid(pl, 256), 256, 0, st>>>(pl->d_n.p, pl->d_off.p, pl->d_poff.p, x_dev, x_dev, nullptr, 0);
  SB_LAUNCH_CHECK_N("sym_ops_kernel");
  return 0;
}

// z = psdinvjmul(xlab, xfrm, y, K):  solve X Z + Z X = 2 Y in the eigenbasis of X   (psdinvjmul.c:101-157)
static int psdinvjmul_core(sb200_psd_plan *pl, const double *xlab_dev, const double *y_dev, double *z_dev);
int sb200_psdinvjmul_dev(sb200_psd_plan *pl, const double *xlab_dev, const double *frms_dev, const double *y_dev, double *z_dev) {
  SB_TRY(ensure_init());
  if (pl->nblk == 0) return 0;
  if (pl->maxn <= PSD_SMALL_MAX && !pl->wy && !pl->wy_rows) {
    // small blocks: two fused congruences.  M = Qb Ys Qb' with the jdiv scaling in its epilogue, then Z = Qb' M Qb
    SB_TRY(build_q(pl, frms_dev, false));
    CongArgs A1{pl->d_Tt.p, y_dev, nullptr, xlab_dev, nullptr, 0, 1, 1, 0, 0, 1};
    SB_TRY(small_congruence(pl, A1, pl->d_Y.p));
    SB_LAUNCH_CHECK_N("small_congruence_kernel");
    CongArgs A2{pl->d_Tt.p, pl->d_Y.p, nullptr, nullptr, nullptr, 0, 0, 0, 0, 0, 1};
    SB_TRY(small_congruence(pl, A2, z_dev));
    SB_LAUNCH_CHECK_N("small_congruence_kernel");
    return 0;
  }
  SB_TRY(build_q(pl, frms_dev));                                      // Q = d_Tt, Q' = d_Wt
  return psdinvjmul_core(pl, xlab_dev, y_dev, z_dev);
}
static int psdinvjmul_core(sb200_psd_plan *pl, const double *xlab_dev, const double *y_dev, double *z_dev) {
  cudaStream_t st = ctx().stream;
  sym_ops_kernel<<<blk_grid(pl, 256), 256, 0, st>>>(pl->d_n.p, pl->d_off.p, pl->d_poff.p, y_dev, pl->d_Y.p, nullptr, 1);   // Ys from tril(Y)
  SB_LAUNCH_CHECK_N("sym_ops_kernel");
  // P = Q Ys           (A = Q, B = Ys symmetric)            -> d_Xp
  gemm_nt_launch(pl->ntiles_full, ctx().sm_count, st, pl->d_desc_full.p, pl->d_tiles_full.p, pl->d_Tt.p, pl->d_Y.p, pl->d_Xp.p, nullptr);
  SB_LAUNCH_CHECK_N("gemm_nt_kernel");
  // M = P Q' (lower)   (A = P, B = Q)                       -> d_Y
  gemm_nt_launch(pl->ntiles_lower, ctx().sm_count, st, pl->d_desc_lower.p, pl->d_tiles_lower.p, pl->d_Xp.p, pl->d_Tt.p, pl->d_Y.p, nullptr);
  SB_LAUNCH_CHECK_N("gemm_nt_kernel");
  sym_ops_kernel<<<blk_grid(pl, 256), 256, 0, st>>>(pl->d_n.p, pl->d_off.p, pl->d_poff.p, pl->d_Y.p, pl->d_Y.p, xlab_dev, 2);
  SB_LAUNCH_CHECK_N("sym_ops_kernel");
  // R = Q' M           (A = Q', B = M symmetric)            -> d_Xp
  gemm_nt_launch(pl->ntiles_full, ctx().sm_count, st, pl->d_desc_full.p, pl->d_tiles_full.p, pl->d_Wt.p, pl->d_Y.p, pl->d_Xp.p, nullptr);
  SB_LAUNCH_CHECK_N("gemm_nt_kernel");
  // Z = R Q (lower)    (A = R, B = Q')                      -> z
  gemm_nt_launch(pl->ntiles_lower, ctx().sm_count, st, pl->d_desc_lower.p, pl->d_tiles_lower.p, pl->d_Xp.p, pl->d_Wt.p, z_dev, nullptr);
  SB_LAUNCH_CHECK_N("gemm_nt_kernel");
  sym_ops_kernel<<<blk_grid(pl, 256), 256, 0, st>>>(pl->d_n.p, pl->d_off.p, pl->d_poff.p, z_dev, z_dev, nullptr, 0);
  SB_LAUNCH_CHECK_N("sym_ops_kernel");
  return 0;
}

int sb200_psdframeit(sb_idx nblk, const sb_idx *n, const double *lab, const double *frms, double *x) {
  sb200_psd_plan *pl = nullptr;
  SB_TRY(sb200_psd_plan_get(&pl, nblk, n));
  if (pl->lenud == 0) return 0;
  arena_reset();
  double *dl = arena<double>((size_t)pl->sumn), *dx = arena<double>((size_t)pl->lenud);
  const double *df = (const double *)mirror_input(frms, sizeof(double) * pl->lenud);      // the frame travels psdinvjmul -> psdframeit x2
  SB_CHECK(dl && df && dx, "psdframeit: out of device memory");
  cudaStream_t st = ctx().stream;
  SB_CUDA(cudaMemcpyAsync(dl, lab, sizeof(double) * pl->sumn, cudaMemcpyHostToDevice, st));
  SB_TRY(sb200_psdframeit_dev(pl, dl, df, dx));
  SB_CUDA(cudaMemcpyAsync(x, dx, sizeof(double) * pl->lenud, cudaMemcpyDeviceToHost, st));
  SB_CUDA(cudaStreamSynchronize(st));
  return 0;
}

int sb200_psdinvjmul(sb_idx nblk, const sb_idx *n, const double *xlab, const double *frms, const double *y, double *z) {
  sb200_psd_plan *pl = nullptr;
  SB_TRY(sb200_psd_plan_get(&pl, nblk, n));
  if (pl->lenud == 0) return 0;
  arena_reset();
  double *dl = arena<double>((size_t)pl->sumn), *dy = arena<double>((size_t)pl->lenud), *dz = arena<double>((size_t)pl->lenud);
  const double *df = (const double *)mirror_input(frms, sizeof(double) * pl->lenud);
  SB_CHECK(dl && df && dy && dz, "psdinvjmul: out of device memory");
  cudaStream_t st = ctx().stream;
  SB_CUDA(cudaMemcpyAsync(dl, xlab, sizeof(double) * pl->sumn, cudaMemcpyHostToDevice, st));
  SB_CUDA(cudaMemcpyAsync(dy, y, sizeof(double) * pl->lenud, cudaMemcpyHostToDevice, st));
  SB_TRY(sb200_psdinvjmul_dev(pl, dl, df, dy, dz));
  SB_CUDA(cudaMemcpyAsync(z, dz, sizeof(double) * pl->lenud, cudaMemcpyDeviceToHost, st));
  SB_CUDA(cudaStreamSynchronize(st));
  return 0;
}


// ---------------------------------------------------------------- Hermitian variants of the host entries
// n[0..nreal) are real symmetric blocks, n[nreal..nblk) Hermitian ones (K.s / K.rsdpN).  Data layout as in
// the reference: real block n^2 doubles, Hermitian block [vec Re; vec Im].  perm: 0-based inside each block.
struct HermCtx {
  sb200_psd_plan *pl = nullptr;        // plan of the embedded orders
  HermBlk *d_blks = nullptr;
  long long raw_len = 0;
  int sumn = 0, maxn = 0, nblk = 0;
  int *d_perm = nullptr;
};
static std::map<Hash128, HermCtx *> g_herm;
static int herm_get(sb_idx nblk, sb_idx nreal, const sb_idx *n, HermCtx **out) {
  SB_TRY(ensure_init());
  SB_CHECK(nreal >= 0 && nreal <= nblk, "number of real PSD blocks out of range");
  Hash128 h = fnv1a(&nblk, sizeof nblk); h = fnv1a(&nreal, sizeof nreal, h); h = fnv1a(n, sizeof(sb_idx) * nblk, h);
  auto it = g_herm.find(h);
  if (it != g_herm.end()) { *out = it->second; return 0; }
  HermCtx *c = new HermCtx();
  std::vector<sb_idx> ne(nblk);
  std::vector<HermBlk> blks(nblk);
  long long raw = 0, emb = 0; int po = 0;
  for (sb_idx k = 0; k < nblk; k++) {
    SB_CHECK(n[k] >= 1 && n[k] < 23170, "PSD block order %lld out of range", (long long)n[k]);
    const int cplx = k >= nreal;
    ne[k] = cplx ? 2 * n[k] : n[k];
    blks[k] = HermBlk{(int)n[k], cplx, po, 0, raw, emb};
    raw += (cplx ? 2 : 1) * n[k] * n[k]; emb += ne[k] * ne[k]; po += (int)n[k];
    c->maxn = std::max(c->maxn, (int)n[k]);
  }
  c->raw_len = raw; c->sumn = po; c->nblk = (int)nblk;
  SB_TRY(sb200_psd_plan_get(&c->pl, nblk, ne.data()));
  SB_CUDA(cudaMalloc(&c->d_blks, sizeof(HermBlk) * std::max<size_t>(blks.size(), 1)));
  SB_CUDA(cudaMemcpy(c->d_blks, blks.data(), sizeof(HermBlk) * blks.size(), cudaMemcpyHostToDevice));
  SB_CUDA(cudaMalloc(&c->d_perm, sizeof(int) * std::max(po, 1)));
  g_herm[h] = c;
  *out = c;
  return 0;
}
static int herm_perm(HermCtx *c, const sb_idx *n, const sb_idx *perm, const int **out) {
  *out = nullptr;
  if (!perm) return 0;
  std::vector<int> p32((size_t)c->sumn);
  int po = 0;
  for (int k = 0; k < c->nblk; k++)
    for (int i = 0; i < n[k]; i++, po++) {
      SB_CHECK(perm[po] >= 0 && perm[po] < n[k], "perm entry out of range in PSD block %d", k);
      p32[po] = (int)perm[po];
    }
  SB_CUDA(cudaMemcpyAsync(c->d_perm, p32.data(), sizeof(int) * p32.size(), cudaMemcpyHostToDevice, ctx().stream));
  SB_CUDA(cudaStreamSynchronize(ctx().stream));
  *out = c->d_perm;
  return 0;
}
static inline dim3 herm_grid(const HermCtx *c) {
  return dim3((unsigned)std::min<long long>(((long long)c->maxn * c->maxn + 255) / 256, 1024), (unsigned)c->nblk);
}

// Y(perm,perm) = U^H U, U = triu(u)   (invcholfac.c:122-160 incl. the prpi branch)
int sb200_invcholfac_h(sb_idx nblk, sb_idx nreal, const sb_idx *n, const double *u, const sb_idx *perm, double *y) {
  HermCtx *c;
  SB_TRY(herm_get(nblk, nreal, n, &c));
  if (c->raw_len == 0) return 0;
  sb200_psd_plan *pl = c->pl;
  arena_reset();
  double *du = arena<double>((size_t)c->raw_len), *dy = arena<double>((size_t)c->raw_len);
  SB_CHECK(du && dy, "invcholfac: out of device memory");
  const int *dperm;
  SB_TRY(herm_perm(c, n, perm, &dperm));
  cudaStream_t st = ctx().stream;
  SB_CUDA(cudaMemcpyAsync(du, u, sizeof(double) * c->raw_len, cudaMemcpyHostToDevice, st));
  herm_embed_kernel<<<herm_grid(c), 256, 0, st>>>(c->d_blks, du, pl->d_Tt.p, nullptr, 1, 1);      // E(U^H)
  SB_LAUNCH_CHECK_N("herm_embed_kernel");
  gemm_nt_launch(pl->ntiles_full, ctx().sm_count, st, pl->d_desc_full.p, pl->d_tiles_full.p, pl->d_Tt.p, pl->d_Tt.p, pl->d_Y.p, nullptr);
  SB_LAUNCH_CHECK_N("gemm_nt_kernel");
  herm_extract_kernel<<<herm_grid(c), 256, 0, st>>>(c->d_blks, pl->d_Y.p, dy, dperm, 1);
  SB_LAUNCH_CHECK_N("herm_extract_kernel");
  SB_CUDA(cudaMemcpyAsync(y, dy, sizeof(double) * c->raw_len, cudaMemcpyDeviceToHost, st));
  SB_CUDA(cudaStreamSynchronize(st));
  return 0;
}

// Y = T^H X T, T = tril(U) / triu(U) (transp), X permuted before (!transp) or Y after (transp)   (psdscale.m:45-119)
int sb200_psdscale_h(sb_idx nblk, sb_idx nreal, const sb_idx *n, const double *u, const sb_idx *perm, const double *x,
                     int transp, double *y) {
  HermCtx *c;
  SB_TRY(herm_get(nblk, nreal, n, &c));
  if (c->raw_len == 0) return 0;
  sb200_psd_plan *pl = c->pl;
  arena_reset();
  double *du = arena<double>((size_t)c->raw_len), *dx = arena<double>((size_t)c->raw_len), *dy = arena<double>((size_t)c->raw_len);
  SB_CHECK(du && dx && dy, "psdscale: out of device memory");
  const int *dperm;
  SB_TRY(herm_perm(c, n, perm, &dperm));
  cudaStream_t st = ctx().stream;
  SB_CUDA(cudaMemcpyAsync(du, u, sizeof(double) * c->raw_len, cudaMemcpyHostToDevice, st));
  SB_CUDA(cudaMemcpyAsync(dx, x, sizeof(double) * c->raw_len, cudaMemcpyHostToDevice, st));
  herm_embed_kernel<<<herm_grid(c), 256, 0, st>>>(c->d_blks, du, pl->d_Tt.p, nullptr, 1, transp ? 1 : 2);       // E(T^H)
  SB_LAUNCH_CHECK_N("herm_embed_kernel");
  herm_embed_kernel<<<herm_grid(c), 256, 0, st>>>(c->d_blks, dx, pl->d_Xp.p, transp ? nullptr : dperm, 0, 0); // E(X(P,P))
  SB_LAUNCH_CHECK_N("herm_embed_kernel");
  // Wt = E(T^H) E(X)' ; Y = E(T^H) Wt' = T^H X T
  gemm_nt_launch(pl->ntiles_full, ctx().sm_count, st, pl->d_desc_full.p, pl->d_tiles_full.p, pl->d_Tt.p, pl->d_Xp.p, pl->d_Wt.p, nullptr);
  SB_LAUNCH_CHECK_N("gemm_nt_kernel");
  gemm_nt_launch(pl->ntiles_full, ctx().sm_count, st, pl->d_desc_full.p, pl->d_tiles_full.p, pl->d_Tt.p, pl->d_Wt.p, pl->d_Y.p, nullptr);
  SB_LAUNCH_CHECK_N("gemm_nt_kernel");
  herm_extract_kernel<<<herm_grid(c), 256, 0, st>>>(c->d_blks, pl->d_Y.p, dy, transp ? dperm : nullptr, 1);
  SB_LAUNCH_CHECK_N("herm_extract_kernel");
  SB_CUDA(cudaMemcpyAsync(y, dy, sizeof(double) * c->raw_len, cudaMemcpyDeviceToHost, st));
  SB_CUDA(cudaStreamSynchronize(st));
  return 0;
}


// Frames of the mixed layout: real block n^2 doubles (last column = beta), Hermitian block 2 n^2 + n
// ([Re c | Im c | beta], psdframeit.c:80-97).  lab: sum(n) eigenvalues.
struct HermFrames { long long *d_fr_off = nullptr; int *d_grp_blk = nullptr, *d_grp_j0 = nullptr; int ngrp = 0; long long fr_len = 0; };
static std::map<HermCtx *, HermFrames *> g_herm_frames;
static int herm_frames_get(HermCtx *c, const sb_idx *n, sb_idx nreal, HermFrames **out) {
  auto it = g_herm_frames.find(c);
  if (it != g_herm_frames.end()) { *out = it->second; return 0; }
  HermFrames *f = new HermFrames();
  std::vector<long long> off(c->nblk);
  std::vector<int> gb, gj;
  long long o = 0;
  for (int k = 0; k < c->nblk; k++) {
    off[k] = o;
    const bool cplx = k >= nreal;
    o += cplx ? 2 * n[k] * n[k] + n[k] : n[k] * n[k];
    if (cplx) for (int j0 = 0; j0 < n[k]; j0 += 8) { gb.push_back(k); gj.push_back(j0); }
  }
  f->fr_len = o; f->ngrp = (int)gb.size();
  SB_CUDA(cudaMalloc(&f->d_fr_off, sizeof(long long) * std::max(c->nblk, 1)));
  SB_CUDA(cudaMemcpy(f->d_fr_off, off.data(), sizeof(long long) * off.size(), cudaMemcpyHostToDevice));
  SB_CUDA(cudaMalloc(&f->d_grp_blk, sizeof(int) * std::max<size_t>(gb.size(), 1)));
  SB_CUDA(cudaMalloc(&f->d_grp_j0, sizeof(int) * std::max<size_t>(gb.size(), 1)));
  if (!gb.empty()) {
    SB_CUDA(cudaMemcpy(f->d_grp_blk, gb.data(), sizeof(int) * gb.size(), cudaMemcpyHostToDevice));
    SB_CUDA(cudaMemcpy(f->d_grp_j0, gj.data(), sizeof(int) * gj.size(), cudaMemcpyHostToDevice));
  }
  g_herm_frames[c] = f;
  *out = f;
  return 0;
}
// Q (embedded) -> pl->d_Tt, Q' -> pl->d_Wt for a mixed real/Hermitian frame vector on the device.
static int herm_build_q(HermCtx *c, HermFrames *f, const double *frms_dev) {
  sb200_psd_plan *pl = c->pl;
  cudaStream_t st = ctx().stream;
  const int maxne = pl->maxn;
  dim3 g((unsigned)std::min<long long>(((long long)maxne * maxne + 255) / 256, 1024), (unsigned)c->nblk);
  herm_frames_kernel<<<g, 256, 0, st>>>(c->d_blks, f->d_fr_off, frms_dev, pl->d_Y.p);
  SB_LAUNCH_CHECK_N("herm_frames_kernel");
  SB_TRY(build_q(pl, pl->d_Y.p));
  if (f->ngrp) {
    householder_q_cplx_kernel<<<f->ngrp, 256, 0, st>>>(c->d_blks, f->d_grp_blk, f->d_grp_j0, f->d_fr_off, frms_dev, pl->d_Tt.p);
    SB_LAUNCH_CHECK_N("householder_q_cplx_kernel");
    int tp = (pl->maxn + 31) / 32;
    transpose_scale_kernel<<<dim3(std::min(1024, tp * tp), pl->nblk), dim3(32, 8), 0, st>>>(pl->d_n.p, pl->d_off.p, pl->d_poff.p, pl->d_Tt.p, nullptr, pl->d_Wt.p);
    SB_LAUNCH_CHECK_N("transpose_scale_kernel");
  }
  return 0;
}
static void herm_lab(const HermCtx *c, const sb_idx *n, sb_idx nreal, const double *lab, std::vector<double> &labe) {
  labe.clear();
  long long po = 0;
  for (int k = 0; k < c->nblk; k++) {
    labe.insert(labe.end(), lab + po, lab + po + n[k]);
    if (k >= nreal) labe.insert(labe.end(), lab + po, lab + po + n[k]);     // E(diag(lab)) = diag(lab, lab)
    po += n[k];
  }
}

// x = psdframeit(lab, frms, K) with Hermitian blocks: X = Qb^H diag(lab) Qb   (psdframeit.c:65-99)
int sb200_psdframeit_h(sb_idx nblk, sb_idx nreal, const sb_idx *n, const double *lab, const double *frms, double *x) {
  HermCtx *c; HermFrames *f;
  SB_TRY(herm_get(nblk, nreal, n, &c));
  if (c->raw_len == 0) return 0;
  SB_TRY(herm_frames_get(c, n, nreal, &f));
  sb200_psd_plan *pl = c->pl;
  std::vector<double> labe;
  herm_lab(c, n, nreal, lab, labe);
  arena_reset();
  double *dl = arena<double>(labe.size()), *df = arena<double>((size_t)f->fr_len), *dxe = arena<double>((size_t)pl->lenud),
         *dx = arena<double>((size_t)c->raw_len);
  SB_CHECK(dl && df && dxe && dx, "psdframeit: out of device memory");
  cudaStream_t st = ctx().stream;
  SB_CUDA(cudaMemcpyAsync(dl, labe.data(), sizeof(double) * labe.size(), cudaMemcpyHostToDevice, st));
  SB_CUDA(cudaMemcpyAsync(df, frms, sizeof(double) * f->fr_len, cudaMemcpyHostToDevice, st));
  SB_TRY(herm_build_q(c, f, df));
  SB_TRY(psdframeit_core(pl, dl, dxe));
  herm_extract_kernel<<<herm_grid(c), 256, 0, st>>>(c->d_blks, dxe, dx, nullptr, 1);
  SB_LAUNCH_CHECK_N("herm_extract_kernel");
  SB_CUDA(cudaMemcpyAsync(x, dx, sizeof(double) * c->raw_len, cudaMemcpyDeviceToHost, st));
  SB_CUDA(cudaStreamSynchronize(st));
  return 0;
}

// z = psdinvjmul(xlab, xfrm, y, K) with Hermitian blocks   (psdinvjmul.c:101-157)
int sb200_psdinvjmul_h(sb_idx nblk, sb_idx nreal, const sb_idx *n, const double *xlab, const double *frms, const double *y, double *z) {
  HermCtx *c; HermFrames *f;
  SB_TRY(herm_get(nblk, nreal, n, &c));
  if (c->raw_len == 0) return 0;
  SB_TRY(herm_frames_get(c, n, nreal, &f));
  sb200_psd_plan *pl = c->pl;
  std::vector<double> labe;
  herm_lab(c, n, nreal, xlab, labe);
  arena_reset();
  double *dl = arena<double>(labe.size()), *df = arena<double>((size_t)f->fr_len), *dye = arena<double>((size_t)pl->lenud),
         *dze = arena<double>((size_t)pl->lenud), *draw = arena<double>((size_t)c->raw_len);
  SB_CHECK(dl && df && dye && dze && draw, "psdinvjmul: out of device memory");
  cudaStream_t st = ctx().stream;
  SB_CUDA(cudaMemcpyAsync(dl, labe.data(), sizeof(double) * labe.size(), cudaMemcpyHostToDevice, st));
  SB_CUDA(cudaMemcpyAsync(df, frms, sizeof(double) * f->fr_len, cudaMemcpyHostToDevice, st));
  SB_CUDA(cudaMemcpyAsync(draw, y, sizeof(double) * c->raw_len, cudaMemcpyHostToDevice, st));
  herm_embed_kernel<<<herm_grid(c), 256, 0, st>>>(c->d_blks, draw, dye, nullptr, 0, 3);       // E(Y), Y completed from its lower triangle
  SB_LAUNCH_CHECK_N("herm_embed_kernel");
  SB_TRY(herm_build_q(c, f, df));
  SB_TRY(psdinvjmul_core(pl, dl, dye, dze));
  herm_extract_kernel<<<herm_grid(c), 256, 0, st>>>(c->d_blks, dze, draw, nullptr, 1);
  SB_LAUNCH_CHECK_N("herm_extract_kernel");
  SB_CUDA(cudaMemcpyAsync(z, draw, sizeof(double) * c->raw_len, cudaMemcpyDeviceToHost, st));
  SB_CUDA(cudaStreamSynchronize(st));
  return 0;
}

}  // extern "C"
