// givens.cu -- urotorder (stable column re-ordering of the triangular PSD scaling factor by Givens
// rotations) and givensrot (apply a stored rotation list to every column of Q).
//
// Reference semantics:
//   urotorder.c:79-180   rotorder: at step k, if max_j u_kj^2 > maxu^2 d_k, bring the column with the
//                        largest remaining norm to position k with Givens rotations (bottom-up),
//                        apply them to the later columns, maintain d by downdating
//   auxgivens.c:43-61    givensrot, :114-140 givensrotuj
//   givensrot.c:60-68    matgivens: for every column, steps k=0..n-2 apply rotations gjc[k]..gjc[k+1]-1
//
// The pivot choices are discrete outputs (perm), so the arithmetic that feeds the comparisons is
// reproduced operation by operation with explicit round-to-nearest intrinsics (no FMA contraction,
// the reference's left-to-right summation order).  Given bit-identical input the outputs are then
// bit-identical to the reference built without FMA (gcc -O2 on x86-64).  Parallelism: one CTA per
// PSD block; inside a step, columns are independent (one thread per column).
#include <algorithm>
#include <map>
#include "sb_internal.h"

namespace sb {

#define DRELTOL 1E-10

__device__ __forceinline__ double mul_(double a, double b) { return __dmul_rn(a, b); }
__device__ __forceinline__ double add_(double a, double b) { return __dadd_rn(a, b); }
__device__ __forceinline__ double sub_(double a, double b) { return __dsub_rn(a, b); }

// auxgivens.c:43-61
__device__ void d_givensrot(double *z, const double *g, int n) {
  double z2 = z[n];
  for (int i = n; i > 0; i--) {
    const double gx = g[2 * (i - 1)], gy = g[2 * (i - 1) + 1];
    const double z1 = z[i - 1];
    z[i] = sub_(mul_(gy, z1), mul_(gx, z2));
    z2 = add_(mul_(gx, z1), mul_(gy, z2));
  }
  z[0] = z2;
}
// auxgivens.c:114-140
__device__ void d_givensrotuj(double *z, const double *g, int n) {
  if (n < 1) return;
  double z2 = z[n - 1];
  z[n] = mul_(z2, g[2 * (n - 1) + 1]);
  z2 = mul_(z2, g[2 * (n - 1)]);
  for (int i = n - 1; i > 0; i--) {
    const double gx = g[2 * (i - 1)], gy = g[2 * (i - 1) + 1];
    const double z1 = z[i - 1];
    z[i] = sub_(mul_(gy, z1), mul_(gx, z2));
    z2 = add_(mul_(gx, z1), mul_(gy, z2));
  }
  z[0] = z2;
}

struct UrotBlk { int n; long long uoff; int poff; long long goff; };   // goff: in doubles, worst-case layout

// ---- speculative "nothing to rotate" pre-pass for large blocks.  The column-pivoting loop below is n dependent steps
// even when no pivot is ever exchanged, which is the common case.  If no exchange happens, every
// decision of the loop depends on the ORIGINAL factor only: d0(i) = sum_{t<=i} u(t,i)^2 (computed once, at k = 0) and
// rowmax(k) = max_{j>k} u(k,j)^2.  Both are computed here in parallel -- d0 with the reference's summation order, so
// the comparisons are the reference's bit for bit -- and the loop is skipped when every test comes out "keep".
static const int UROT_PRECHECK_MIN_N = 128;
__global__ void urot_colnorm_kernel(const UrotBlk *blks, const double *W, double *d_all) {
  const UrotBlk B = blks[blockIdx.y];
  const int n = B.n, i = blockIdx.x * blockDim.x + threadIdx.x;
  if (n < UROT_PRECHECK_MIN_N || i >= n) return;
  const double *x = W + B.uoff + (long long)i * n;
  double sacc = 0.0;
  for (int t = 0; t <= i; t++) sacc = add_(sacc, mul_(x[t], x[t]));
  d_all[B.poff + i] = sacc;
}
__global__ void __launch_bounds__(256) urot_rowmax_kernel(const UrotBlk *blks, const double *W, double *g_all) {
  const UrotBlk B = blks[blockIdx.y];
  const int n = B.n;
  if (n < UROT_PRECHECK_MIN_N || blockIdx.x * 32 >= n) return;
  __shared__ double sh[8][32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, k = blockIdx.x * 32 + lane;
  const double *u = W + B.uoff;
  double mx = 0.0;
  for (int j = blockIdx.x * 32 + 1 + warp; j < n; j += 8)
    if (k < n && j > k) { const double v = u[k + (long long)j * n]; mx = fmax(mx, mul_(v, v)); }
  sh[warp][lane] = mx;
  __syncthreads();
  if (warp == 0 && k < n) {
    for (int w = 1; w < 8; w++) mx = fmax(mx, sh[w][lane]);
    g_all[B.goff + k] = mx;                            // parked in the (still unused) rotation area
  }
}

__global__ void __launch_bounds__(256)
urotorder_kernel(const UrotBlk *blks, double *W, int *perm_all, int *gjc_all, double *g_all, double *d_all,
                 double maxusqr) {
  const UrotBlk B = blks[blockIdx.x];
  const int n = B.n;
  double *u = W + B.uoff;
  int *perm = perm_all + B.poff, *gjc = gjc_all + B.poff;
  double *d = d_all + B.poff;
  double *g = g_all + B.goff;
  __shared__ double s_h, s_red[32];
  __shared__ int s_flag, s_pivk, s_inz, s_redi[32];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nw = blockDim.x >> 5;
  for (int j = tid; j < n; j += blockDim.x) perm[j] = j;
  if (n >= UROT_PRECHECK_MIN_N) {                      // the pre-pass left d0 in d and rowmax in g
    const double h0 = mul_(d[0], DRELTOL);
    int keep = 1;
    for (int k = tid; k < n - 1; k += blockDim.x) {
      const double dk = d[k];
      if (k >= 1 && dk <= h0) keep = 0;                 // the loop would recompute the norms here
      if (g[k] > mul_(maxusqr, dk)) keep = 0;           // the loop would exchange a pivot here
    }
    keep = __syncthreads_and(keep);
    if (keep) {
      for (int k = tid; k < n; k += blockDim.x) { gjc[k] = 0; g[k] = 0.0; }       // (un-park rowmax: the rotation area stays clean)
      return;
    }
  }
  if (n >= UROT_PRECHECK_MIN_N) for (int k = tid; k < n; k += blockDim.x) g[k] = 0.0;
  __syncthreads();
  if (tid == 0) { d[0] = 0.0; s_h = 1.0; s_pivk = 0; s_inz = 0; }
  __syncthreads();
  for (int k = 0; k < n - 1; k++) {
    double *rowuk = u + k;
    __syncthreads();                                 // everyone is done with last step's flags
    if (tid == 0) { gjc[k] = s_inz; s_flag = (d[perm[k]] <= s_h); }
    __syncthreads();
    if (s_flag) {                                    // d(i) = sum(u(k:j,i).^2) from scratch
      for (int j = k + tid; j < n; j += blockDim.x) {
        const int i = perm[j];
        const double *x = rowuk + (long long)i * n;
        double s = 0.0;
        for (int t = 0; t < j + 1 - k; t++) s = add_(s, mul_(x[t], x[t]));
        d[i] = s;
      }
      __syncthreads();
      if (tid == 0) s_h = mul_(d[perm[k]], DRELTOL);
    }
    // ukmax = max U(k,perm(k+1:n)).^2
    double mx = 0.0;
    for (int j = k + 1 + tid; j < n; j += blockDim.x) {
      double v = rowuk[(long long)perm[j] * n];
      v = mul_(v, v);
      mx = fmax(mx, v);
    }
    for (int o = 16; o > 0; o >>= 1) mx = fmax(mx, __shfl_down_sync(0xffffffffu, mx, o));
    if (lane == 0) s_red[warp] = mx;
    __syncthreads();
    if (tid == 0) {
      for (int w = 1; w < nw; w++) mx = fmax(mx, s_red[w]);
      s_flag = (mx > mul_(maxusqr, d[perm[k]]));
    }
    __syncthreads();
    if (!s_flag) continue;                           // uniform
    // best pivot: first j in k+1..n-1 with the largest d(perm(j)) (strict >, so ties keep the first)
    double bd = 0.0; int bj = 0x7fffffff;
    for (int j = k + 1 + tid; j < n; j += blockDim.x) {
      double v = d[perm[j]];
      if (v > bd || (v == bd && v > 0.0 && j < bj)) { bd = v; bj = j; }
    }
    for (int o = 16; o > 0; o >>= 1) {
      double ov = __shfl_down_sync(0xffffffffu, bd, o); int oj = __shfl_down_sync(0xffffffffu, bj, o);
      if (ov > bd || (ov == bd && ov > 0.0 && oj < bj)) { bd = ov; bj = oj; }
    }
    __syncthreads();
    if (lane == 0) { s_red[warp] = bd; s_redi[warp] = bj; }
    __syncthreads();
    if (tid == 0) {
      for (int w = 1; w < nw; w++)
        if (s_red[w] > bd || (s_red[w] == bd && bd > 0.0 && s_redi[w] < bj)) { bd = s_red[w]; bj = s_redi[w]; }
      if (bd > 0.0) s_pivk = bj;                     // else: keep the previous pivk like the reference
      const int pivk = s_pivk, m = pivk - k;
      const int j = perm[pivk];
      double *uj = rowuk + (long long)j * n;
      double *gk = g + 2 * (long long)s_inz;
      double nexty = uj[m];
      double y = mul_(nexty, nexty);
      for (int i = m; i > 0; i--) {
        double gx = uj[i - 1], gy = nexty;
        y = add_(y, mul_(gx, gx));
        nexty = sqrt(y);
        gk[2 * (i - 1)] = gx / nexty;
        gk[2 * (i - 1) + 1] = gy / nexty;
      }
      uj[0] = nexty;
      for (int t = pivk; t > k; t--) perm[t] = perm[t - 1];
      perm[k] = j;
    }
    __syncthreads();
    {
      const int m = s_pivk - k;
      const double *gk = g + 2 * (long long)s_inz;
      for (int i = 1 + tid; k + i < n; i += blockDim.x) {
        double *z = rowuk + (long long)perm[k + i] * n;
        if (i <= m) d_givensrotuj(z, gk, i);
        else d_givensrot(z, gk, m);
      }
      __syncthreads();
      for (int j = k + 1 + tid; j < n; j += blockDim.x) {
        const int i = perm[j];
        const double x = rowuk[(long long)i * n];
        d[i] = sub_(d[i], mul_(x, x));
      }
      if (tid == 0) s_inz += m;
    }
    __syncthreads();
  }
  if (tid == 0) gjc[n - 1] = s_inz;
}

// u_out(i,j) = W(i, perm[j]) for i <= j, mirrored below (uperm + triu2sym, sdmauxTriu.c:90-100,136-145)
__global__ void uperm_sym_kernel(const UrotBlk *blks, const double *W, const int *perm_all, double *uout) {
  const UrotBlk B = blks[blockIdx.y];
  const int n = B.n;
  const int *perm = perm_all + B.poff;
  const long long tot = (long long)n * n;
  for (long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x; idx < tot; idx += (long long)gridDim.x * blockDim.x) {
    int i = (int)(idx % n), j = (int)(idx / n);
    int lo = min(i, j), hi = max(i, j);
    uout[B.uoff + idx] = W[B.uoff + lo + (long long)perm[hi] * n];
  }
}

// givensrot.c:60-68: every column of every block, steps k = 0..n-2
__global__ void matgivens_kernel(const UrotBlk *blks, const int *gjc_all, const double *g_all, double *y) {
  const UrotBlk B = blks[blockIdx.y];
  const int n = B.n;
  const int *gjc = gjc_all + B.poff;
  const double *g = g_all + B.goff;
  for (int j = blockIdx.x * blockDim.x + threadIdx.x; j < n; j += gridDim.x * blockDim.x) {
    double *col = y + B.uoff + (long long)j * n;
    for (int k = 0; k < n - 1; k++) {
      const int m = gjc[k + 1] - gjc[k];
      if (m > 0) d_givensrot(col + k, g + 2 * (long long)gjc[k], m);
    }
  }
}

// ---------------------------------------------------------------- Hermitian blocks (urotorder.c:197-304, auxgivens.c:62-205)
// Same algorithm on [Re U | Im U] with rotations [conj(x), y; y, -x] stored as (Re x, Im x, y); the arithmetic is
// restated operation by operation (explicit round-to-nearest, the reference's association) for bit-identical output.
__device__ void d_prpigivensrot(double *z, double *zi, const double *g, int n) {
  double z2 = z[n], z2im = zi[n];
  for (int i = n; i > 0; i--) {
    const double gx = g[3 * (i - 1)], gxim = g[3 * (i - 1) + 1], gy = g[3 * (i - 1) + 2];
    const double z1 = z[i - 1], z1im = zi[i - 1];
    z[i] = add_(sub_(mul_(gy, z1), mul_(gx, z2)), mul_(gxim, z2im));
    zi[i] = sub_(sub_(mul_(gy, z1im), mul_(gx, z2im)), mul_(gxim, z2));
    const double n2 = add_(add_(mul_(gx, z1), mul_(gxim, z1im)), mul_(gy, z2));
    const double n2im = add_(sub_(mul_(gx, z1im), mul_(gxim, z1)), mul_(gy, z2im));
    z2 = n2; z2im = n2im;
  }
  z[0] = z2; zi[0] = z2im;
}
__device__ void d_prpigivensrotuj(double *z, double *zi, const double *g, int n) {
  if (n < 1) return;
  double z2 = z[n - 1];
  z[n] = mul_(z2, g[3 * (n - 1) + 2]);
  double z2im = mul_(-z2, g[3 * (n - 1) + 1]);
  z2 = mul_(z2, g[3 * (n - 1)]);
  for (int i = n - 1; i > 0; i--) {
    const double gx = g[3 * (i - 1)], gxim = g[3 * (i - 1) + 1], gy = g[3 * (i - 1) + 2];
    const double z1 = z[i - 1], z1im = zi[i - 1];
    z[i] = add_(sub_(mul_(gy, z1), mul_(gx, z2)), mul_(gxim, z2im));
    zi[i] = sub_(sub_(mul_(gy, z1im), mul_(gx, z2im)), mul_(gxim, z2));
    const double n2 = add_(add_(mul_(gx, z1), mul_(gxim, z1im)), mul_(gy, z2));
    const double n2im = add_(sub_(mul_(gx, z1im), mul_(gxim, z1)), mul_(gy, z2im));
    z2 = n2; z2im = n2im;
  }
  z[0] = z2; zi[0] = z2im;
}

__global__ void __launch_bounds__(256)
urotorder_cplx_kernel(const UrotBlk *blks, double *W, int *perm_all, int *gjc_all, double *g_all, double *d_all,
                      double maxusqr) {
  const UrotBlk B = blks[blockIdx.x];
  const int n = B.n;
  double *u = W + B.uoff, *upi = u + (long long)n * n;
  int *perm = perm_all + B.poff, *gjc = gjc_all + B.poff;
  double *d = d_all + B.poff;
  double *g = g_all + B.goff;
  __shared__ double s_h, s_red[32];
  __shared__ int s_flag, s_pivk, s_inz, s_redi[32];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nw = blockDim.x >> 5;
  for (int j = tid; j < n; j += blockDim.x) perm[j] = j;
  if (tid == 0) { d[0] = 0.0; s_h = 1.0; s_pivk = 0; s_inz = 0; }
  __syncthreads();
  for (int k = 0; k < n - 1; k++) {
    double *rowuk = u + k, *rowukpi = upi + k;
    __syncthreads();
    if (tid == 0) { gjc[k] = s_inz; s_flag = (d[perm[k]] <= s_h); }
    __syncthreads();
    if (s_flag) {                                    // d(i) = |u(k:j,i)|^2 from scratch (the diagonal u(j,i) is real)
      for (int j = k + tid; j < n; j += blockDim.x) {
        const int i = perm[j];
        const double *x = rowuk + (long long)i * n, *xi = rowukpi + (long long)i * n;
        double sr = 0.0, si = 0.0;
        for (int t = 0; t < j + 1 - k; t++) sr = add_(sr, mul_(x[t], x[t]));
        for (int t = 0; t < j - k; t++) si = add_(si, mul_(xi[t], xi[t]));
        d[i] = add_(sr, si);
      }
      __syncthreads();
      if (tid == 0) s_h = mul_(d[perm[k]], DRELTOL);
    }
    double mx = 0.0;
    for (int j = k + 1 + tid; j < n; j += blockDim.x) {
      const double a = rowuk[(long long)perm[j] * n], b = rowukpi[(long long)perm[j] * n];
      mx = fmax(mx, add_(mul_(a, a), mul_(b, b)));
    }
    for (int o = 16; o > 0; o >>= 1) mx = fmax(mx, __shfl_down_sync(0xffffffffu, mx, o));
    if (lane == 0) s_red[warp] = mx;
    __syncthreads();
    if (tid == 0) {
      for (int w = 1; w < nw; w++) mx = fmax(mx, s_red[w]);
      s_flag = (mx > mul_(maxusqr, d[perm[k]]));
    }
    __syncthreads();
    if (!s_flag) continue;                           // uniform
    double bd = 0.0; int bj = 0x7fffffff;
    for (int j = k + 1 + tid; j < n; j += blockDim.x) {
      double v = d[perm[j]];
      if (v > bd || (v == bd && v > 0.0 && j < bj)) { bd = v; bj = j; }
    }
    for (int o = 16; o > 0; o >>= 1) {
      double ov = __shfl_down_sync(0xffffffffu, bd, o); int oj = __shfl_down_sync(0xffffffffu, bj, o);
      if (ov > bd || (ov == bd && ov > 0.0 && oj < bj)) { bd = ov; bj = oj; }
    }
    __syncthreads();
    if (lane == 0) { s_red[warp] = bd; s_redi[warp] = bj; }
    __syncthreads();
    if (tid == 0) {
      for (int w = 1; w < nw; w++)
        if (s_red[w] > bd || (s_red[w] == bd && bd > 0.0 && s_redi[w] < bj)) { bd = s_red[w]; bj = s_redi[w]; }
      if (bd > 0.0) s_pivk = bj;
      const int pivk = s_pivk, m = pivk - k;
      const int j = perm[pivk];
      double *uj = rowuk + (long long)j * n, *ujpi = rowukpi + (long long)j * n;
      double *gk = g + 3 * (long long)s_inz;
      double nexty = uj[m];
      double y = mul_(nexty, nexty);
      for (int i = m; i > 0; i--) {
        const double gx = uj[i - 1], gxim = ujpi[i - 1], gy = nexty;
        y = add_(y, add_(mul_(gx, gx), mul_(gxim, gxim)));
        nexty = sqrt(y);
        gk[3 * (i - 1)] = gx / nexty;
        gk[3 * (i - 1) + 1] = gxim / nexty;
        gk[3 * (i - 1) + 2] = gy / nexty;
      }
      uj[0] = nexty;
      for (int t = pivk; t > k; t--) perm[t] = perm[t - 1];
      perm[k] = j;
    }
    __syncthreads();
    {
      const int m = s_pivk - k;
      const double *gk = g + 3 * (long long)s_inz;
      for (int i = 1 + tid; k + i < n; i += blockDim.x) {
        double *z = rowuk + (long long)perm[k + i] * n, *zi = rowukpi + (long long)perm[k + i] * n;
        if (i <= m) d_prpigivensrotuj(z, zi, gk, i);
        else d_prpigivensrot(z, zi, gk, m);
      }
      __syncthreads();
      for (int j = k + 1 + tid; j < n; j += blockDim.x) {
        const int i = perm[j];
        const double x = rowuk[(long long)i * n], xi = rowukpi[(long long)i * n];
        d[i] = sub_(d[i], add_(mul_(x, x), mul_(xi, xi)));
      }
      if (tid == 0) s_inz += m;
    }
    __syncthreads();
  }
  if (tid == 0) gjc[n - 1] = s_inz;
}

// uperm + triu2herm: Re symmetric, Im skew-symmetric with zero diagonal (sdmauxTriu.c:108-145)
__global__ void uperm_herm_kernel(const UrotBlk *blks, const double *W, const int *perm_all, double *uout) {
  const UrotBlk B = blks[blockIdx.y];
  const int n = B.n;
  const int *perm = perm_all + B.poff;
  const long long tot = (long long)n * n;
  for (long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x; idx < tot; idx += (long long)gridDim.x * blockDim.x) {
    int i = (int)(idx % n), j = (int)(idx / n);
    int lo = min(i, j), hi = max(i, j);
    const long long src = B.uoff + lo + (long long)perm[hi] * n;
    uout[B.uoff + idx] = W[src];
    const double im = W[src + tot];
    uout[B.uoff + tot + idx] = (i == j) ? 0.0 : (i < j ? im : -im);
  }
}

__global__ void matgivens_cplx_kernel(const UrotBlk *blks, const int *gjc_all, const double *g_all, double *y) {
  const UrotBlk B = blks[blockIdx.y];
  const int n = B.n;
  const int *gjc = gjc_all + B.poff;
  const double *g = g_all + B.goff;
  for (int j = blockIdx.x * blockDim.x + threadIdx.x; j < n; j += gridDim.x * blockDim.x) {
    double *col = y + B.uoff + (long long)j * n, *coli = col + (long long)n * n;
    for (int k = 0; k < n - 1; k++) {
      const int m = gjc[k + 1] - gjc[k];
      if (m > 0) d_prpigivensrot(col + k, coli + k, g + 3 * (long long)gjc[k], m);
    }
  }
}

}  // namespace sb
using namespace sb;

static int make_blocks(sb_idx nblk, const sb_idx *n, std::vector<UrotBlk> &blks, long long &lenud, long long &sumn, long long &gtot) {
  lenud = 0; sumn = 0; gtot = 0;
  for (sb_idx k = 0; k < nblk; k++) {
    SB_CHECK(n[k] >= 1 && n[k] < 46340, "PSD block order out of range");
    UrotBlk b; b.n = (int)n[k]; b.uoff = lenud; b.poff = (int)sumn; b.goff = gtot;
    blks.push_back(b);
    lenud += n[k] * n[k]; sumn += n[k]; gtot += n[k] * (n[k] - 1);     // 2 doubles per rotation, n(n-1)/2 rotations
  }
  return 0;
}

// Block descriptors on the device, worst-case rotation layout; cached per block-size list so that the
// *_dev entries can be recorded into a CUDA graph (no allocation or copy at call time after the first).
static std::map<Hash128, UrotBlk *> g_blk_cache;
static int device_blocks(sb_idx nblk, const sb_idx *n, UrotBlk **out, long long &lenud, long long &sumn, long long &gtot, int &maxn) {
  std::vector<UrotBlk> blks;
  SB_TRY(make_blocks(nblk, n, blks, lenud, sumn, gtot));
  maxn = 0; for (auto &b : blks) maxn = std::max(maxn, b.n);
  Hash128 h = fnv1a(&nblk, sizeof nblk); h = fnv1a(n, sizeof(sb_idx) * nblk, h);
  auto it = g_blk_cache.find(h);
  if (it != g_blk_cache.end()) { *out = it->second; return 0; }
  UrotBlk *d = nullptr;
  SB_CUDA(cudaMalloc(&d, sizeof(UrotBlk) * std::max<size_t>(blks.size(), 1)));
  SB_CUDA(cudaMemcpy(d, blks.data(), sizeof(UrotBlk) * blks.size(), cudaMemcpyHostToDevice));
  g_blk_cache[h] = d;
  *out = d;
  return 0;
}

extern "C" {

// Device-resident urotorder.  u_dev is read, work_dev (lenud + sum n doubles) is scratch; outputs:
// u_out_dev (lenud), perm_dev / gjc_dev (sum n ints: 0-based inside each block / cumulative rotation
// counts), g_dev in the worst-case layout (block k at sum_{j<k} n_j(n_j-1) doubles).
int sb200_urotorder_dev(sb_idx nblk, const sb_idx *n, const double *u_dev, double maxu, double *u_out_dev,
                        int *perm_dev, int *gjc_dev, double *g_dev, double *work_dev) {
  SB_TRY(ensure_init());
  UrotBlk *db; long long lenud, sumn, gtot; int maxn;
  SB_TRY(device_blocks(nblk, n, &db, lenud, sumn, gtot, maxn));
  if (lenud == 0) return 0;
  cudaStream_t st = ctx().stream;
  double *W = work_dev, *d = work_dev + lenud;
  SB_CUDA(cudaMemcpyAsync(W, u_dev, sizeof(double) * lenud, cudaMemcpyDeviceToDevice, st));
  if (gtot) SB_CUDA(cudaMemsetAsync(g_dev, 0, sizeof(double) * gtot, st));
  SB_CUDA(cudaMemsetAsync(gjc_dev, 0, sizeof(int) * sumn, st));
  if (maxn >= UROT_PRECHECK_MIN_N) {
    urot_colnorm_kernel<<<dim3((unsigned)((maxn + 127) / 128), (unsigned)nblk), 128, 0, st>>>(db, W, d);
    SB_LAUNCH_CHECK_N("urot_colnorm_kernel");
    urot_rowmax_kernel<<<dim3((unsigned)((maxn + 31) / 32), (unsigned)nblk), 256, 0, st>>>(db, W, g_dev);
    SB_LAUNCH_CHECK_N("urot_rowmax_kernel");
  }
  urotorder_kernel<<<(unsigned)nblk, 256, 0, st>>>(db, W, perm_dev, gjc_dev, g_dev, d, maxu * maxu);
  SB_LAUNCH_CHECK_N("urotorder_kernel");
  uperm_sym_kernel<<<dim3((unsigned)std::min<long long>(((long long)maxn * maxn + 255) / 256, 1024), (unsigned)nblk), 256, 0, st>>>(db, W, perm_dev, u_out_dev);
  SB_LAUNCH_CHECK_N("uperm_sym_kernel");
  return 0;
}

// Device-resident givensrot on the outputs of sb200_urotorder_dev (worst-case rotation layout).
// y_dev may alias x_dev.
int sb200_givensrot_dev(sb_idx nblk, const sb_idx *n, const int *gjc_dev, const double *g_dev, const double *x_dev,
                        double *y_dev) {
  SB_TRY(ensure_init());
  UrotBlk *db; long long lenud, sumn, gtot; int maxn;
  SB_TRY(device_blocks(nblk, n, &db, lenud, sumn, gtot, maxn));
  if (lenud == 0) return 0;
  cudaStream_t st = ctx().stream;
  if (y_dev != x_dev) SB_CUDA(cudaMemcpyAsync(y_dev, x_dev, sizeof(double) * lenud, cudaMemcpyDeviceToDevice, st));
  matgivens_kernel<<<dim3((unsigned)((maxn + 127) / 128), (unsigned)nblk), 128, 0, st>>>(db, gjc_dev, g_dev, y_dev);
  SB_LAUNCH_CHECK_N("matgivens_kernel");
  return 0;
}

// [u,perm,gjc,g] = urotorder(u,K,maxu): host entry.  perm_out: 0-based inside each block (the stub
// composes it with permIN); gjc_out: per block n_k entries (gjc[n_k-1] = number of rotations);
// g_out: rotations of block k start at g_out + goff[k] (worst-case layout n_k(n_k-1) doubles per block).
int sb200_urotorder(sb_idx nblk, const sb_idx *n, const double *u, double maxu, double *u_out, sb_idx *perm_out,
                    sb_idx *gjc_out, double *g_out) {
  SB_TRY(ensure_init());
  std::vector<UrotBlk> blks;
  long long lenud, sumn, gtot;
  SB_TRY(make_blocks(nblk, n, blks, lenud, sumn, gtot));
  if (lenud == 0) return 0;
  arena_reset();
  UrotBlk *db = arena<UrotBlk>(blks.size());
  double *W = arena<double>(lenud), *uo = arena<double>(lenud), *g = arena<double>(std::max<long long>(gtot, 1)), *d = arena<double>(sumn);
  int *perm = arena<int>(sumn), *gjc = arena<int>(sumn);
  SB_CHECK(db && W && uo && g && d && perm && gjc, "urotorder: out of device memory");
  cudaStream_t st = ctx().stream;
  SB_CUDA(cudaMemcpyAsync(db, blks.data(), sizeof(UrotBlk) * blks.size(), cudaMemcpyHostToDevice, st));
  SB_CUDA(cudaMemcpyAsync(W, u, sizeof(double) * lenud, cudaMemcpyHostToDevice, st));
  SB_CUDA(cudaMemsetAsync(g, 0, sizeof(double) * std::max<long long>(gtot, 1), st));
  SB_CUDA(cudaMemsetAsync(gjc, 0, sizeof(int) * sumn, st));
  int maxn = 0; for (auto &b : blks) maxn = std::max(maxn, b.n);
  if (maxn >= UROT_PRECHECK_MIN_N) {
    urot_colnorm_kernel<<<dim3((unsigned)((maxn + 127) / 128), (unsigned)nblk), 128, 0, st>>>(db, W, d);
    SB_LAUNCH_CHECK_N("urot_colnorm_kernel");
    urot_rowmax_kernel<<<dim3((unsigned)((maxn + 31) / 32), (unsigned)nblk), 256, 0, st>>>(db, W, g);
    SB_LAUNCH_CHECK_N("urot_rowmax_kernel");
  }
  urotorder_kernel<<<(unsigned)nblk, 256, 0, st>>>(db, W, perm, gjc, g, d, maxu * maxu);
  SB_LAUNCH_CHECK_N("urotorder_kernel");
  uperm_sym_kernel<<<dim3((unsigned)std::min<long long>(((long long)maxn * maxn + 255) / 256, 1024), (unsigned)nblk), 256, 0, st>>>(db, W, perm, uo);
  SB_LAUNCH_CHECK_N("uperm_sym_kernel");
  std::vector<int> hp(sumn), hg(sumn);
  SB_CUDA(cudaMemcpyAsync(u_out, uo, sizeof(double) * lenud, cudaMemcpyDeviceToHost, st));
  SB_CUDA(cudaMemcpyAsync(hp.data(), perm, sizeof(int) * sumn, cudaMemcpyDeviceToHost, st));
  SB_CUDA(cudaMemcpyAsync(hg.data(), gjc, sizeof(int) * sumn, cudaMemcpyDeviceToHost, st));
  if (gtot) SB_CUDA(cudaMemcpyAsync(g_out, g, sizeof(double) * gtot, cudaMemcpyDeviceToHost, st));
  SB_CUDA(cudaStreamSynchronize(st));
  for (long long i = 0; i < sumn; i++) { perm_out[i] = hp[i]; gjc_out[i] = hg[i]; }
  return 0;
}

// y = givensrot(gjc,g,x,K): gjc per block (n_k entries, 0-based counts); g packed per block: the
// rotations of block k start right after those of block k-1 (2 doubles each).
int sb200_givensrot(sb_idx nblk, const sb_idx *n, const sb_idx *gjc, const double *g, sb_idx glen, const double *x, double *y) {
  SB_TRY(ensure_init());
  std::vector<UrotBlk> blks;
  long long lenud, sumn, gtot;
  SB_TRY(make_blocks(nblk, n, blks, lenud, sumn, gtot));
  if (lenud == 0) return 0;
  long long inz = 0;
  std::vector<int> g32(sumn);
  for (auto &b : blks) {
    b.goff = inz;
    for (int i = 0; i < b.n; i++) {
      sb_idx v = gjc[b.poff + i];
      SB_CHECK(v >= 0 && v <= (sb_idx)b.n * (b.n - 1) / 2 && (i == 0 || v >= gjc[b.poff + i - 1]), "givensrot: gjc is not a valid rotation count list");
      g32[b.poff + i] = (int)v;
    }
    inz += 2 * gjc[b.poff + b.n - 1];
    SB_CHECK(inz <= glen, "g size mismatch");
  }
  arena_reset();
  UrotBlk *db = arena<UrotBlk>(blks.size());
  double *dy = arena<double>(lenud), *dg = arena<double>(std::max<long long>(inz, 1));
  int *dgjc = arena<int>(sumn);
  SB_CHECK(db && dy && dg && dgjc, "givensrot: out of device memory");
  cudaStream_t st = ctx().stream;
  SB_CUDA(cudaMemcpyAsync(db, blks.data(), sizeof(UrotBlk) * blks.size(), cudaMemcpyHostToDevice, st));
  SB_CUDA(cudaMemcpyAsync(dy, x, sizeof(double) * lenud, cudaMemcpyHostToDevice, st));
  SB_CUDA(cudaMemcpyAsync(dgjc, g32.data(), sizeof(int) * sumn, cudaMemcpyHostToDevice, st));
  if (inz) SB_CUDA(cudaMemcpyAsync(dg, g, sizeof(double) * inz, cudaMemcpyHostToDevice, st));
  int maxn = 0; for (auto &b : blks) maxn = std::max(maxn, b.n);
  matgivens_kernel<<<dim3((unsigned)((maxn + 127) / 128), (unsigned)nblk), 128, 0, st>>>(db, dgjc, dg, dy);
  SB_LAUNCH_CHECK_N("matgivens_kernel");
  SB_CUDA(cudaMemcpyAsync(y, dy, sizeof(double) * lenud, cudaMemcpyDeviceToHost, st));
  SB_CUDA(cudaStreamSynchronize(st));
  return 0;
}


// ---- mixed real / Hermitian blocks (blocks [nreal, nblk) Hermitian: u = [vec Re; vec Im], rotations 3 doubles)
static int make_blocks_h(sb_idx nblk, sb_idx nreal, const sb_idx *n, std::vector<UrotBlk> &blks, long long &lenud, long long &sumn, long long &gtot) {
  lenud = 0; sumn = 0; gtot = 0;
  SB_CHECK(nreal >= 0 && nreal <= nblk, "number of real PSD blocks out of range");
  for (sb_idx k = 0; k < nblk; k++) {
    SB_CHECK(n[k] >= 1 && n[k] < 32768, "PSD block order out of range");
    const bool cplx = k >= nreal;
    UrotBlk b; b.n = (int)n[k]; b.uoff = lenud; b.poff = (int)sumn; b.goff = gtot;
    blks.push_back(b);
    lenud += (cplx ? 2 : 1) * n[k] * n[k]; sumn += n[k];
    gtot += cplx ? 3 * n[k] * (n[k] - 1) / 2 : n[k] * (n[k] - 1);
  }
  return 0;
}

// g_out: worst-case layout, block k at sum_{j<k} (real: n_j(n_j-1), Hermitian: 3 n_j(n_j-1)/2) doubles.
int sb200_urotorder_h(sb_idx nblk, sb_idx nreal, const sb_idx *n, const double *u, double maxu, double *u_out,
                      sb_idx *perm_out, sb_idx *gjc_out, double *g_out) {
  SB_TRY(ensure_init());
  std::vector<UrotBlk> blks;
  long long lenud, sumn, gtot;
  SB_TRY(make_blocks_h(nblk, nreal, n, blks, lenud, sumn, gtot));
  if (lenud == 0) return 0;
  arena_reset();
  UrotBlk *db = arena<UrotBlk>(blks.size());
  double *W = arena<double>(lenud), *uo = arena<double>(lenud), *g = arena<double>(std::max<long long>(gtot, 1)), *d = arena<double>(sumn);
  int *perm = arena<int>(sumn), *gjc = arena<int>(sumn);
  SB_CHECK(db && W && uo && g && d && perm && gjc, "urotorder: out of device memory");
  cudaStream_t st = ctx().stream;
  SB_CUDA(cudaMemcpyAsync(db, blks.data(), sizeof(UrotBlk) * blks.size(), cudaMemcpyHostToDevice, st));
  SB_CUDA(cudaMemcpyAsync(W, u, sizeof(double) * lenud, cudaMemcpyHostToDevice, st));
  SB_CUDA(cudaMemsetAsync(g, 0, sizeof(double) * std::max<long long>(gtot, 1), st));
  SB_CUDA(cudaMemsetAsync(gjc, 0, sizeof(int) * sumn, st));
  int maxr = 0, maxc = 0;
  for (sb_idx k = 0; k < nblk; k++) (k < nreal ? maxr : maxc) = std::max(k < nreal ? maxr : maxc, (int)n[k]);
  if (nreal > 0) {
    int maxn = 0; for (sb_idx k2 = 0; k2 < nreal; k2++) maxn = std::max(maxn, blks[k2].n);
    if (maxn >= UROT_PRECHECK_MIN_N) {
      urot_colnorm_kernel<<<dim3((unsigned)((maxn + 127) / 128), (unsigned)nreal), 128, 0, st>>>(db, W, d);
      SB_LAUNCH_CHECK_N("urot_colnorm_kernel");
      urot_rowmax_kernel<<<dim3((unsigned)((maxn + 31) / 32), (unsigned)nreal), 256, 0, st>>>(db, W, g);
      SB_LAUNCH_CHECK_N("urot_rowmax_kernel");
    }
    urotorder_kernel<<<(unsigned)nreal, 256, 0, st>>>(db, W, perm, gjc, g, d, maxu * maxu);
    SB_LAUNCH_CHECK_N("urotorder_kernel");
    uperm_sym_kernel<<<dim3((unsigned)std::min<long long>(((long long)maxr * maxr + 255) / 256, 1024), (unsigned)nreal), 256, 0, st>>>(db, W, perm, uo);
    SB_LAUNCH_CHECK_N("uperm_sym_kernel");
  }
  if (nblk > nreal) {
    urotorder_cplx_kernel<<<(unsigned)(nblk - nreal), 256, 0, st>>>(db + nreal, W, perm, gjc, g, d, maxu * maxu);
    SB_LAUNCH_CHECK_N("urotorder_cplx_kernel");
    uperm_herm_kernel<<<dim3((unsigned)std::min<long long>(((long long)maxc * maxc + 255) / 256, 1024), (unsigned)(nblk - nreal)), 256, 0, st>>>(db + nreal, W, perm, uo);
    SB_LAUNCH_CHECK_N("uperm_herm_kernel");
  }
  std::vector<int> hp(sumn), hg(sumn);
  SB_CUDA(cudaMemcpyAsync(u_out, uo, sizeof(double) * lenud, cudaMemcpyDeviceToHost, st));
  SB_CUDA(cudaMemcpyAsync(hp.data(), perm, sizeof(int) * sumn, cudaMemcpyDeviceToHost, st));
  SB_CUDA(cudaMemcpyAsync(hg.data(), gjc, sizeof(int) * sumn, cudaMemcpyDeviceToHost, st));
  if (gtot) SB_CUDA(cudaMemcpyAsync(g_out, g, sizeof(double) * gtot, cudaMemcpyDeviceToHost, st));
  SB_CUDA(cudaStreamSynchronize(st));
  for (long long i = 0; i < sumn; i++) { perm_out[i] = hp[i]; gjc_out[i] = hg[i]; }
  return 0;
}

// g packed: the rotations of block k follow those of block k-1 (2 doubles each for real, 3 for Hermitian blocks).
int sb200_givensrot_h(sb_idx nblk, sb_idx nreal, const sb_idx *n, const sb_idx *gjc, const double *g, sb_idx glen,
                      const double *x, double *y) {
  SB_TRY(ensure_init());
  std::vector<UrotBlk> blks;
  long long lenud, sumn, gtot;
  SB_TRY(make_blocks_h(nblk, nreal, n, blks, lenud, sumn, gtot));
  if (lenud == 0) return 0;
  long long inz = 0;
  std::vector<int> g32(sumn);
  int maxr = 0, maxc = 0;
  for (sb_idx k = 0; k < nblk; k++) {
    UrotBlk &b = blks[k];
    b.goff = inz;
    for (int i = 0; i < b.n; i++) {
      sb_idx v = gjc[b.poff + i];
      SB_CHECK(v >= 0 && v <= (sb_idx)b.n * (b.n - 1) / 2 && (i == 0 || v >= gjc[b.poff + i - 1]), "givensrot: gjc is not a valid rotation count list");
      g32[b.poff + i] = (int)v;
    }
    inz += (k < nreal ? 2 : 3) * gjc[b.poff + b.n - 1];
    SB_CHECK(inz <= glen, "g size mismatch");
    (k < nreal ? maxr : maxc) = std::max(k < nreal ? maxr : maxc, b.n);
  }
  arena_reset();
  UrotBlk *db = arena<UrotBlk>(blks.size());
  double *dy = arena<double>(lenud), *dg = arena<double>(std::max<long long>(inz, 1));
  int *dgjc = arena<int>(sumn);
  SB_CHECK(db && dy && dg && dgjc, "givensrot: out of device memory");
  cudaStream_t st = ctx().stream;
  SB_CUDA(cudaMemcpyAsync(db, blks.data(), sizeof(UrotBlk) * blks.size(), cudaMemcpyHostToDevice, st));
  SB_CUDA(cudaMemcpyAsync(dy, x, sizeof(double) * lenud, cudaMemcpyHostToDevice, st));
  SB_CUDA(cudaMemcpyAsync(dgjc, g32.data(), sizeof(int) * sumn, cudaMemcpyHostToDevice, st));
  if (inz) SB_CUDA(cudaMemcpyAsync(dg, g, sizeof(double) * inz, cudaMemcpyHostToDevice, st));
  if (nreal > 0) {
    matgivens_kernel<<<dim3((unsigned)((maxr + 127) / 128), (unsigned)nreal), 128, 0, st>>>(db, dgjc, dg, dy);
    SB_LAUNCH_CHECK_N("matgivens_kernel");
  }
  if (nblk > nreal) {
    matgivens_cplx_kernel<<<dim3((unsigned)((maxc + 127) / 128), (unsigned)(nblk - nreal)), 128, 0, st>>>(db + nreal, dgjc, dg, dy);
    SB_LAUNCH_CHECK_N("matgivens_cplx_kernel");
  }
  SB_CUDA(cudaMemcpyAsync(y, dy, sizeof(double) * lenud, cudaMemcpyDeviceToHost, st));
  SB_CUDA(cudaStreamSynchronize(st));
  return 0;
}

}  // extern "C"
