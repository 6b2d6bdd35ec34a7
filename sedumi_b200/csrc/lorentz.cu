// lorentz.cu -- streaming Lorentz-cone kernels: ddot, qblkmul, quadadd.
//
// Reference semantics:
//   ddot.c:69-76      dense:  y(k,col) = d[k]' * x[k,col] for every Lorentz block k
//   ddot.c:95-155     sparse: y(k,j) for every block k in which column j of X has nonzeros
//   qblkmul.c:110-115 y[k] = mu(k) * d[k]
//   quadadd.c:58-81   error-free (double-double) accumulation (zhi,zlo) = (xhi,xlo) + y
// All three are pure HBM streams (SURVEY.md section 8d): one pass, coalesced, grid-stride.
#include <algorithm>
#include "sb_internal.h"

namespace sb {

// a group of G lanes per (block, column): dot over the block's rows.  G follows the average cone length so that short
// cones do not pay a 5-step shuffle reduction for two elements per lane.
template <int G>
__global__ void ddot_dense_kernel(int nblk, const long long *bs, const double *d, const double *X, long long ldx,
                                  long long ncol, double *y) {
  const int gl = threadIdx.x % G;
  long long w = (blockIdx.x * (long long)blockDim.x + threadIdx.x) / G;
  const long long nw = ((long long)gridDim.x * blockDim.x) / G;
  const long long tot = (long long)nblk * ncol;
  const unsigned lane = threadIdx.x & 31;
  const unsigned gmask = G == 32 ? 0xffffffffu : (((1u << G) - 1u) << (lane / G * G));
  for (; w < tot; w += nw) {
    const int k = (int)(w % nblk);
    const long long col = w / nblk;
    const double *x = X + col * ldx;
    double acc = 0.0;
    for (long long i = bs[k] + gl; i < bs[k + 1]; i += G) acc += d[i] * x[i];
#pragma unroll
    for (int o = G / 2; o > 0; o >>= 1) acc += __shfl_down_sync(gmask, acc, o, G);
    if (gl == 0) y[w] = acc;
  }
}

// one thread per output entry: segment [seg[e], seg[e+1]) of X's nonzeros, all inside one block
__global__ void ddot_sparse_kernel(long long nout, const long long *seg_lo, const long long *seg_hi, const int *xir,
                                   const double *xpr, const double *d, long long d_shift, double *y) {
  for (long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x; e < nout; e += (long long)gridDim.x * blockDim.x) {
    double acc = 0.0;
    for (long long p = seg_lo[e]; p < seg_hi[e]; p++) acc += d[xir[p] - d_shift] * xpr[p];
    y[e] = acc;
  }
}

// y[k] = mu(k) * d[k].  Long cones: a warp per cone (mu read once, coalesced stream).  Short cones: every thread takes
// 4 consecutive elements, finds its cone once by bisection and walks forward from there (the first version bisected
// per element: 20 dependent loads for 2^20 cones, 15 % of the HBM peak).
__global__ void qblkmul_warp_kernel(int nblk, const long long *bs, const double *mu, const double *d, double *y) {
  const int lane = threadIdx.x & 31;
  long long w = (blockIdx.x * (long long)blockDim.x + threadIdx.x) >> 5;
  const long long nw = ((long long)gridDim.x * blockDim.x) >> 5;
  for (; w < nblk; w += nw) {
    const double m = mu[w];
    for (long long i = bs[w] + lane; i < bs[w + 1]; i += 32) y[i] = m * d[i];
  }
}
__global__ void qblkmul_chunk_kernel(int nblk, const long long *bs, const double *mu, const double *d, double *y) {
  const long long tot = bs[nblk];
  for (long long i0 = 4 * (blockIdx.x * (long long)blockDim.x + threadIdx.x); i0 < tot; i0 += 4 * (long long)gridDim.x * blockDim.x) {
    int l = 0, h = nblk;
    while (h - l > 1) { int mid = (l + h) >> 1; if (bs[mid] <= i0) l = mid; else h = mid; }
    long long nxt = bs[l + 1];
    double m = mu[l];
    const long long i1 = min(i0 + 4, tot);
    for (long long i = i0; i < i1; i++) {
      while (i >= nxt) { l++; nxt = bs[l + 1]; m = mu[l]; }
      y[i] = m * d[i];
    }
  }
}

// Branch-exact restatement of rquaddadd (quadadd.c:58-81); explicit _rn intrinsics so the
// compiler can neither contract nor reassociate the error-free transformation.
__global__ void quadadd_kernel(long long n, const double *xhi, const double *xlo, const double *y, double *zhi, double *zlo) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    double a = xhi[i], b = xlo[i], c = y[i], hi, lo;
    if (fabs(c) > fabs(a)) {
      hi = __dadd_rn(c, a);
      a = __dsub_rn(a, __dsub_rn(hi, c));
      lo = __dadd_rn(b, a);
    } else {
      double t = __dadd_rn(b, c);
      b = __dsub_rn(b, __dsub_rn(t, c));
      hi = __dadd_rn(a, t);
      t = __dsub_rn(t, __dsub_rn(hi, a));
      lo = __dadd_rn(b, t);
    }
    zhi[i] = hi; zlo[i] = lo;
  }
}

static inline unsigned grid_for(long long n, int per = 256) {
  long long g = (n + per - 1) / per;
  long long cap = (long long)ctx().sm_count * 16;
  return (unsigned)std::max<long long>(1, std::min(g, cap));
}

}  // namespace sb
using namespace sb;

extern "C" {

// ---- device-resident variants
int sb200_ddot_dense_dev(sb_idx nblk, const long long *bs_dev, const double *d_dev, const double *X_dev, sb_idx ldx,
                         sb_idx ncol, double *y_dev) {
  SB_TRY(ensure_init());
  if (nblk == 0 || ncol == 0) return 0;
  // average cone length decides the lanes per cone; the host entry and the callers pass ldx = the norm-bound length
  const long long avg = nblk > 0 ? (long long)ldx / nblk : 0;
  if (avg >= 256) ddot_dense_kernel<32><<<grid_for(nblk * ncol * 32), 256, 0, ctx().stream>>>((int)nblk, bs_dev, d_dev, X_dev, ldx, ncol, y_dev);
  else if (avg >= 24) ddot_dense_kernel<8><<<grid_for(nblk * ncol * 8), 256, 0, ctx().stream>>>((int)nblk, bs_dev, d_dev, X_dev, ldx, ncol, y_dev);
  else ddot_dense_kernel<2><<<grid_for(nblk * ncol * 2), 256, 0, ctx().stream>>>((int)nblk, bs_dev, d_dev, X_dev, ldx, ncol, y_dev);
  SB_LAUNCH_CHECK_N("ddot_dense_kernel");
  return 0;
}
int sb200_qblkmul_dev(sb_idx nblk, const long long *bs_dev, sb_idx qdim, const double *mu_dev, const double *d_dev, double *y_dev) {
  SB_TRY(ensure_init());
  if (qdim == 0) return 0;
  if (nblk > 0 && qdim / nblk >= 48) qblkmul_warp_kernel<<<grid_for(nblk * 32), 256, 0, ctx().stream>>>((int)nblk, bs_dev, mu_dev, d_dev, y_dev);
  else qblkmul_chunk_kernel<<<grid_for((qdim + 3) / 4), 256, 0, ctx().stream>>>((int)nblk, bs_dev, mu_dev, d_dev, y_dev);
  SB_LAUNCH_CHECK_N("qblkmul_kernel");
  return 0;
}
int sb200_quadadd_dev(sb_idx n, const double *xhi, const double *xlo, const double *y, double *zhi, double *zlo) {
  SB_TRY(ensure_init());
  if (n == 0) return 0;
  quadadd_kernel<<<grid_for(n), 256, 0, ctx().stream>>>(n, xhi, xlo, y, zhi, zlo);
  SB_LAUNCH_CHECK_N("quadadd_kernel");
  return 0;
}

// ---- host entries
// bs[0..nblk]: 0-based block starts RELATIVE to the first norm-bound row (bs[0]=0).
// d: qdim values; X: first norm-bound row of column 0, leading dimension ldx.
int sb200_ddot_dense(sb_idx nblk, const sb_idx *bs, const double *d, const double *X, sb_idx ldx, sb_idx ncol, double *y) {
  SB_TRY(ensure_init());
  if (nblk == 0 || ncol == 0) return 0;
  arena_reset();
  const sb_idx qdim = bs[nblk];
  std::vector<long long> b64(bs, bs + nblk + 1);
  long long *dbs = arena<long long>(nblk + 1);
  double *dd = arena<double>((size_t)qdim), *dX = arena<double>((size_t)(qdim * ncol)), *dy = arena<double>((size_t)(nblk * ncol));
  SB_CHECK(dbs && dd && dX && dy, "ddot: out of device memory");
  cudaStream_t st = ctx().stream;
  SB_CUDA(cudaMemcpyAsync(dbs, b64.data(), sizeof(long long) * (nblk + 1), cudaMemcpyHostToDevice, st));
  SB_CUDA(cudaMemcpyAsync(dd, d, sizeof(double) * qdim, cudaMemcpyHostToDevice, st));
  SB_CUDA(cudaMemcpy2DAsync(dX, sizeof(double) * qdim, X, sizeof(double) * ldx, sizeof(double) * qdim, (size_t)ncol, cudaMemcpyHostToDevice, st));
  SB_TRY(sb200_ddot_dense_dev(nblk, dbs, dd, dX, qdim, ncol, dy));
  SB_CUDA(cudaMemcpyAsync(y, dy, sizeof(double) * nblk * ncol, cudaMemcpyDeviceToHost, st));
  SB_CUDA(cudaStreamSynchronize(st));
  return 0;
}

// Sparse X (CSC, m columns): per column j the nonzeros in [xlo[j], xhi[j]) lie in the Lorentz
// norm-bound rows [bs_abs[0], bs_abs[nblk]).  Output pattern (yjc, yir) and values ypr are written;
// yir/ypr need room for sum(xhi-xlo) entries.  Returns the number of entries in *nnz_out.
int sb200_ddot_sparse(sb_idx nblk, const sb_idx *bs_abs, const double *d, sb_idx m, const sb_idx *xlo, const sb_idx *xhi,
                      const sb_idx *xir, const double *xpr, sb_idx *yjc, sb_idx *yir, double *ypr, sb_idx *nnz_out) {
  SB_TRY(ensure_init());
  // structural pass on the host: one output entry per (column, touched block)
  std::vector<long long> seg_lo, seg_hi;
  sb_idx knz = 0;
  sb_idx pmin = -1, pmax = 0;
  const sb_idx lend = bs_abs[nblk];
  for (sb_idx j = 0; j < m; j++) {
    yjc[j] = knz;
    sb_idx p = xlo[j];
    while (p < xhi[j] && xir[p] < lend) {
      sb_idx i = xir[p];
      SB_CHECK(i >= bs_abs[0], "ddot: X nonzero below the Lorentz norm-bound rows");
      sb_idx k = (sb_idx)(std::upper_bound(bs_abs, bs_abs + nblk + 1, i) - bs_abs) - 1;
      sb_idx p0 = p;
      while (p < xhi[j] && xir[p] < bs_abs[k + 1]) p++;
      seg_lo.push_back(p0); seg_hi.push_back(p);
      yir[knz++] = k;
      if (pmin < 0) pmin = p0;
      pmax = p;
    }
  }
  yjc[m] = knz;
  *nnz_out = knz;
  if (knz == 0) return 0;
  arena_reset();
  const sb_idx span = pmax - pmin;
  for (auto &v : seg_lo) v -= pmin;
  for (auto &v : seg_hi) v -= pmin;
  std::vector<int> ir32((size_t)span);
  for (sb_idx p = 0; p < span; p++) ir32[p] = (int)xir[pmin + p];
  const sb_idx qdim = bs_abs[nblk] - bs_abs[0];
  long long *dlo = arena<long long>(knz), *dhi = arena<long long>(knz);
  int *dir = arena<int>(span);
  double *dpr = arena<double>(span), *dd = arena<double>(qdim), *dy = arena<double>(knz);
  SB_CHECK(dlo && dhi && dir && dpr && dd && dy, "ddot: out of device memory");
  cudaStream_t st = ctx().stream;
  SB_CUDA(cudaMemcpyAsync(dlo, seg_lo.data(), sizeof(long long) * knz, cudaMemcpyHostToDevice, st));
  SB_CUDA(cudaMemcpyAsync(dhi, seg_hi.data(), sizeof(long long) * knz, cudaMemcpyHostToDevice, st));
  SB_CUDA(cudaMemcpyAsync(dir, ir32.data(), sizeof(int) * span, cudaMemcpyHostToDevice, st));
  SB_CUDA(cudaMemcpyAsync(dpr, xpr + pmin, sizeof(double) * span, cudaMemcpyHostToDevice, st));
  SB_CUDA(cudaMemcpyAsync(dd, d, sizeof(double) * qdim, cudaMemcpyHostToDevice, st));
  ddot_sparse_kernel<<<grid_for(knz), 256, 0, st>>>(knz, dlo, dhi, dir, dpr, dd, bs_abs[0], dy);
  SB_LAUNCH_CHECK_N("ddot_sparse_kernel");
  SB_CUDA(cudaMemcpyAsync(ypr, dy, sizeof(double) * knz, cudaMemcpyDeviceToHost, st));
  SB_CUDA(cudaStreamSynchronize(st));
  return 0;
}

int sb200_qblkmul(sb_idx nblk, const sb_idx *bs, const double *mu, const double *d, double *y) {
  SB_TRY(ensure_init());
  const sb_idx qdim = bs[nblk];
  if (qdim == 0) return 0;
  arena_reset();
  std::vector<long long> b64(bs, bs + nblk + 1);
  long long *dbs = arena<long long>(nblk + 1);
  double *dmu = arena<double>(nblk), *dd = arena<double>(qdim), *dy = arena<double>(qdim);
  SB_CHECK(dbs && dmu && dd && dy, "qblkmul: out of device memory");
  cudaStream_t st = ctx().stream;
  SB_CUDA(cudaMemcpyAsync(dbs, b64.data(), sizeof(long long) * (nblk + 1), cudaMemcpyHostToDevice, st));
  SB_CUDA(cudaMemcpyAsync(dmu, mu, sizeof(double) * nblk, cudaMemcpyHostToDevice, st));
  SB_CUDA(cudaMemcpyAsync(dd, d, sizeof(double) * qdim, cudaMemcpyHostToDevice, st));
  SB_TRY(sb200_qblkmul_dev(nblk, dbs, qdim, dmu, dd, dy));
  SB_CUDA(cudaMemcpyAsync(y, dy, sizeof(double) * qdim, cudaMemcpyDeviceToHost, st));
  SB_CUDA(cudaStreamSynchronize(st));
  return 0;
}

int sb200_quadadd(sb_idx n, const double *xhi, const double *xlo, const double *y, double *zhi, double *zlo) {
  SB_TRY(ensure_init());
  if (n == 0) return 0;
  arena_reset();
  double *a = arena<double>(n), *b = arena<double>(n), *c = arena<double>(n), *h = arena<double>(n), *l = arena<double>(n);
  SB_CHECK(a && b && c && h && l, "quadadd: out of device memory");
  cudaStream_t st = ctx().stream;
  SB_CUDA(cudaMemcpyAsync(a, xhi, sizeof(double) * n, cudaMemcpyHostToDevice, st));
  SB_CUDA(cudaMemcpyAsync(b, xlo, sizeof(double) * n, cudaMemcpyHostToDevice, st));
  SB_CUDA(cudaMemcpyAsync(c, y, sizeof(double) * n, cudaMemcpyHostToDevice, st));
  SB_TRY(sb200_quadadd_dev(n, a, b, c, h, l));
  SB_CUDA(cudaMemcpyAsync(zhi, h, sizeof(double) * n, cudaMemcpyDeviceToHost, st));
  SB_CUDA(cudaMemcpyAsync(zlo, l, sizeof(double) * n, cudaMemcpyDeviceToHost, st));
  SB_CUDA(cudaStreamSynchronize(st));
  return 0;
}

}  // extern "C"

// ------------------------------------------------------------------------------------------------
// adendotd / adenscale: dense Lorentz blocks (adendotd.c:69-126, adenscale.c:62-77).
namespace sb {
// One CTA per dense Lorentz block k.  Ad(:,k) on the pattern of Ablk(:,k) =
//   adotd(:,k) + d1[q_k] * aden(:,k) + sum_{dense norm-bound columns j of block k} d2[col_j] * aden2(:,j)
__global__ void __launch_bounds__(256)
adendotd_kernel(int m, const long long *adjc, const int *adir, double *adpr, const long long *sjc, const int *sir,
                const double *spr, const long long *ajc, const int *air, const double *apr, int nq, const double *d1q,
                const int *colbeg, const double *d2c, double *fwork) {
  const int k = blockIdx.x;
  double *f = fwork + (long long)k * m;
  for (long long i = adjc[k] + threadIdx.x; i < adjc[k + 1]; i += blockDim.x) f[adir[i]] = 0.0;
  __syncthreads();
  for (long long i = sjc[k] + threadIdx.x; i < sjc[k + 1]; i += blockDim.x) f[sir[i]] = spr[i];
  __syncthreads();
  const double dj = d1q[k];
  for (long long i = ajc[k] + threadIdx.x; i < ajc[k + 1]; i += blockDim.x) f[air[i]] += dj * apr[i];
  __syncthreads();
  for (int j = colbeg[k]; j < colbeg[k + 1]; j++) {            // dense norm-bound columns of this block
    const double w = d2c[j];
    for (long long i = ajc[nq + j] + threadIdx.x; i < ajc[nq + j + 1]; i += blockDim.x) f[air[i]] += w * apr[i];
    __syncthreads();
  }
  for (long long i = adjc[k] + threadIdx.x; i < adjc[k + 1]; i += blockDim.x) adpr[i] = f[adir[i]];
}
}  // namespace sb

extern "C" {

// Ad = adendotd(dense,d,sparAd,Ablk,blkstart).  aden = dense.A(:, nl+1:end) as CSC over nq+nden columns
// (ajc relative to its own start), d1q[k] = d.q1(dense.q(k)), colbeg[k..k+1] = range of dense norm-bound
// columns belonging to block k, d2c[j] = d.q2 entry of dense column j.
int sb200_adendotd(sb_idx m, sb_idx nq, sb_idx nden, const sb_idx *adjc, const sb_idx *adir, const sb_idx *sjc, const sb_idx *sir,
                   const double *spr, const sb_idx *ajc, const sb_idx *air, const double *apr, const double *d1q,
                   const sb_idx *colbeg, const double *d2c, double *adpr) {
  SB_TRY(ensure_init());
  if (nq == 0) return 0;
  arena_reset();
  cudaStream_t st = ctx().stream;
  const sb_idx nad = adjc[nq], ns = sjc[nq], na = ajc[nq + nden];
  std::vector<long long> j1(adjc, adjc + nq + 1), j2(sjc, sjc + nq + 1), j3(ajc, ajc + nq + nden + 1);
  std::vector<int> i1, i2, i3, cb(nq + 1);
  SB_TRY(to_i32(adir, nad, i1, "Ablk.ir")); SB_TRY(to_i32(sir, ns, i2, "sparAd.ir")); SB_TRY(to_i32(air, na, i3, "dense.A.ir"));
  for (sb_idx k = 0; k <= nq; k++) cb[k] = (int)colbeg[k];
  long long *dj1 = arena<long long>(nq + 1), *dj2 = arena<long long>(nq + 1), *dj3 = arena<long long>(nq + nden + 1);
  int *di1 = arena<int>(std::max<sb_idx>(nad, 1)), *di2 = arena<int>(std::max<sb_idx>(ns, 1)), *di3 = arena<int>(std::max<sb_idx>(na, 1)), *dcb = arena<int>(nq + 1);
  double *dsp = arena<double>(std::max<sb_idx>(ns, 1)), *dap = arena<double>(std::max<sb_idx>(na, 1)), *dd1 = arena<double>(nq),
         *dd2 = arena<double>(std::max<sb_idx>(nden, 1)), *dad = arena<double>(std::max<sb_idx>(nad, 1)), *df = arena<double>(m * nq);
  SB_CHECK(dj1 && dj2 && dj3 && di1 && di2 && di3 && dcb && dsp && dap && dd1 && dd2 && dad && df, "adendotd: out of device memory");
  SB_CUDA(cudaMemcpyAsync(dj1, j1.data(), sizeof(long long) * (nq + 1), cudaMemcpyHostToDevice, st));
  SB_CUDA(cudaMemcpyAsync(dj2, j2.data(), sizeof(long long) * (nq + 1), cudaMemcpyHostToDevice, st));
  SB_CUDA(cudaMemcpyAsync(dj3, j3.data(), sizeof(long long) * (nq + nden + 1), cudaMemcpyHostToDevice, st));
  if (nad) SB_CUDA(cudaMemcpyAsync(di1, i1.data(), sizeof(int) * nad, cudaMemcpyHostToDevice, st));
  if (ns) { SB_CUDA(cudaMemcpyAsync(di2, i2.data(), sizeof(int) * ns, cudaMemcpyHostToDevice, st)); SB_CUDA(cudaMemcpyAsync(dsp, spr, sizeof(double) * ns, cudaMemcpyHostToDevice, st)); }
  if (na) { SB_CUDA(cudaMemcpyAsync(di3, i3.data(), sizeof(int) * na, cudaMemcpyHostToDevice, st)); SB_CUDA(cudaMemcpyAsync(dap, apr, sizeof(double) * na, cudaMemcpyHostToDevice, st)); }
  SB_CUDA(cudaMemcpyAsync(dcb, cb.data(), sizeof(int) * (nq + 1), cudaMemcpyHostToDevice, st));
  SB_CUDA(cudaMemcpyAsync(dd1, d1q, sizeof(double) * nq, cudaMemcpyHostToDevice, st));
  if (nden) SB_CUDA(cudaMemcpyAsync(dd2, d2c, sizeof(double) * nden, cudaMemcpyHostToDevice, st));
  adendotd_kernel<<<(unsigned)nq, 256, 0, st>>>((int)m, dj1, di1, dad, dj2, di2, dsp, dj3, di3, dap, (int)nq, dd1, dcb, dd2, df);
  SB_LAUNCH_CHECK_N("adendotd_kernel");
  if (nad) SB_CUDA(cudaMemcpyAsync(adpr, dad, sizeof(double) * nad, cudaMemcpyDeviceToHost, st));
  SB_CUDA(cudaStreamSynchronize(st));
  return 0;
}

}  // extern "C"
