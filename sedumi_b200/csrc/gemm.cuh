// gemm.cuh -- batched FP64 "NT" GEMM engine used by the PSD-cone kernels.
//
//   C(i,c) (+)= alpha * sum_k A(i,k) * B(c,k)          A: M x K, B: N x K, both column-major
//
// so both operands are read contiguously along the output index (coalesced tile loads).
// A column gather on A (A(i,k) = A[i + gather[k]*lda]) serves getada3's D(:,R) operand;
// triangular hints let tiles skip the k-ranges that are structurally zero (U'U, T'XT).
// One flattened tile list drives a whole batch of independent products in one launch
// (per-PSD-block / per-constraint problems of different sizes), so the grid scales with
// the total work, not with the number of problems.
//
// FP64 on sm_90a has no wgmma kind; the tensor path for doubles is the legacy
// mma.sync m8n8k4 DMMA, used by the 64x64 tile kernel below (each warp owns a 32x32
// sub-tile = 4x4 DMMA fragments).  Operands are staged through shared memory.
#pragma once
#include <cuda_runtime.h>

namespace sb {

enum { TRI_NONE = 0, TRI_K_LE_ROW = 1, TRI_K_GE_ROW = 2 };   // nonzero only where k <= row / k >= row

// Operands are addressed as base pointer (kernel argument) + offset (descriptor), so the
// descriptor/tile arrays depend only on the cone structure and live in a plan.
struct GemmDesc {
  long long offA; long long gatherOff; int lda; int a_tri;   // gatherOff < 0: no column gather
  long long offB; int ldb; int b_tri;
  long long offC; int ldc;
  int M, N, K;
  int lower;        // 1: only entries with i >= c are needed (tiles strictly above are skipped)
  int accumulate;   // 0: C = alpha*AB ; 1: C += alpha*AB
  double alpha;
};
struct GemmTile { int prob, ti, tj; };

static const int GT = 64;     // tile edge
static const int GK = 16;     // k-slab
static const int GST = 3;     // cp.async pipeline depth (52 KB per CTA: four 128-thread CTAs per SM, the register limit)
static const int GEMM_SMEM = GST * 2 * GK * (GT + 4) * 8;     // dynamic shared memory per tile CTA
// threads per tile: 128 * KG (KG k-groups of 4 warps; each warp owns a 32x32 sub-tile = 4x4 DMMA fragments)

__device__ __forceinline__ void dmma_m8n8k4(double &c0, double &c1, double a, double b) {
  asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};\n"
               : "+d"(c0), "+d"(c1) : "d"(a), "d"(b));
}

__device__ __forceinline__ void cp_async_8(void *smem, const void *gmem, int src_bytes) {   // src_bytes 0: zero-fill
  const unsigned sa = (unsigned)__cvta_generic_to_shared(smem);
  asm volatile("cp.async.ca.shared.global [%0], [%1], 8, %2;\n" :: "r"(sa), "l"(gmem), "r"(src_bytes) : "memory");
}
__device__ __forceinline__ void cp_async_16(void *smem, const void *gmem) {
  const unsigned sa = (unsigned)__cvta_generic_to_shared(smem);
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;\n" :: "r"(sa), "l"(gmem) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;\n" ::: "memory"); }
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_group 0;\n" ::: "memory"); }
template <int N> __device__ __forceinline__ void cp_async_wait_group() { asm volatile("cp.async.wait_group %0;\n" ::"n"(N) : "memory"); }

// One operand slab (64 rows x GK k-values) global -> shared, element (i, kk) -> S[kk][i].
// Fast path: 16-byte copies, no predicates (interior tile, k-slab fully inside the nonzero range,
// even leading dimension and 16-byte aligned base).  General path: 8-byte copies, zero-filled where
// the element is out of range or structurally zero.
template <int KG, int GKT>
__device__ __forceinline__ void gemm_stage_slab(double (*S)[GT + 4], const double *g, int ld, int rows, int r0, int K, int k0,
                                                int tri, const int *gather, bool vec_ok) {
  const int tid = threadIdx.x;
  // rows of the tile no fragment reads (beyond the last 8-row fragment with entries of C) are not staged at all
  const int rows8 = min(GT, ((rows - r0 + 7) >> 3) << 3);
  bool fast = vec_ok && ((rows & 1) == 0) && (k0 + GKT <= K);
  if (tri == TRI_K_LE_ROW) fast = fast && (k0 + GKT - 1 <= r0);
  if (tri == TRI_K_GE_ROW) fast = fast && (k0 >= r0 + GT - 1);
  if (fast) {
    const int i = (tid & 31) * 2;
    if (i < rows8) {
      const unsigned nbytes = (r0 + i < rows) ? 16u : 0u;         // rows is even: a 16-byte chunk is inside or outside as a whole
#pragma unroll
      for (int r = 0; r < GKT / (4 * KG); r++) {
        const int kk = (tid >> 5) + 4 * KG * r, k = k0 + kk;
        const long long col = gather ? gather[k] : k;
        const unsigned sa = (unsigned)__cvta_generic_to_shared(&S[kk][i]);
        asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;\n" :: "r"(sa), "l"(nbytes ? g + r0 + i + col * ld : g), "r"(nbytes) : "memory");
      }
    }
  } else {
    const int i = tid & 63, gi = r0 + i;
    if (i < rows8) {
#pragma unroll
      for (int r = 0; r < GKT / (2 * KG); r++) {
        const int kk = (tid >> 6) + 2 * KG * r, k = k0 + kk;
        bool nz = (k < K) && (gi < rows);
        if (tri == TRI_K_LE_ROW) nz = nz && (k <= gi);
        if (tri == TRI_K_GE_ROW) nz = nz && (k >= gi);
        const double *src = g;
        if (nz) src = g + gi + (long long)(gather ? gather[k] : k) * ld;
        cp_async_8(&S[kk][i], src, nz ? 8 : 0);
      }
    }
  }
}

// DMMAs of one k-slab on a warp's sub-tile: NRA x NCB fragments (DIAG: the lower triangle of NRA x NRA), straight-line code
template <int KG, int GKT, int NRA, int NCB, bool DIAG>
__device__ __forceinline__ void gemm_warp_mma_static(double (&acc)[4][4][2], const double (*As)[GT + 4], const double (*Bs)[GT + 4],
                                                     int wr, int wc, int qr, int qc, int kgrp) {
#pragma unroll
  for (int kq = 0; kq < GKT; kq += 4 * KG) {
    const int k4 = kq + 4 * kgrp;
    double af[4], bf[4];
#pragma unroll
    for (int a = 0; a < NRA; a++) af[a] = As[k4 + qc][wr + 8 * a + qr];     // A frag: row = lane/4, k = lane%4
#pragma unroll
    for (int b = 0; b < NCB; b++) bf[b] = Bs[k4 + qc][wc + 8 * b + qr];     // B frag: k = lane%4, col = lane/4
#pragma unroll
    for (int a = 0; a < NRA; a++)
#pragma unroll
      for (int b = 0; b < NCB; b++)
        if (!DIAG || a >= b) dmma_m8n8k4(acc[a][b][0], acc[a][b][1], af[a], bf[b]);
  }
}
template <int KG, int GKT>
__device__ __forceinline__ void gemm_warp_mma(double (&acc)[4][4][2], const double (*As)[GT + 4], const double (*Bs)[GT + 4],
                                              int wr, int wc, int qr, int qc, int kgrp, int variant) {
#define SB_GEMM_CASE(v, NRA, NCB, DG) case v: gemm_warp_mma_static<KG, GKT, NRA, NCB, DG>(acc, As, Bs, wr, wc, qr, qc, kgrp); break;
  switch (variant) {
    SB_GEMM_CASE(15, 4, 4, false) SB_GEMM_CASE(19, 4, 4, true)
    SB_GEMM_CASE(0, 1, 1, false) SB_GEMM_CASE(1, 1, 2, false) SB_GEMM_CASE(2, 1, 3, false) SB_GEMM_CASE(3, 1, 4, false)
    SB_GEMM_CASE(4, 2, 1, false) SB_GEMM_CASE(5, 2, 2, false) SB_GEMM_CASE(6, 2, 3, false) SB_GEMM_CASE(7, 2, 4, false)
    SB_GEMM_CASE(8, 3, 1, false) SB_GEMM_CASE(9, 3, 2, false) SB_GEMM_CASE(10, 3, 3, false) SB_GEMM_CASE(11, 3, 4, false)
    SB_GEMM_CASE(12, 4, 1, false) SB_GEMM_CASE(13, 4, 2, false) SB_GEMM_CASE(14, 4, 3, false)
    SB_GEMM_CASE(16, 1, 1, true) SB_GEMM_CASE(17, 2, 2, true) SB_GEMM_CASE(18, 3, 3, true)
    default: break;
  }
#undef SB_GEMM_CASE
}

// KG = 2: 256 threads = 2 k-groups x 4 warps; warp w owns rows [32*(w&1), +32) x cols [32*((w>>1)&1), +32) of the
// tile (16 DMMAs per 8 shared-memory fragment loads) and, inside every k-slab, the k4-steps of its
// k-group (w>>2); the two partial tiles are added through shared memory at the end.  Splitting k inside
// the CTA keeps 8 warps busy per tile: the per-block products here often have fewer tiles than the GPU
// has SMs (n = 1000: 256 tiles, against 132 SMs; 4 warps per tile leave most warp slots empty).
// KG = 1 (128 threads, no split) is used when a launch has tiles to spare: more CTAs per SM.
// GST-stage cp.async pipeline: slabs s+1..s+GST-1 are in flight while the DMMAs of slab s run (with two
// stages the copy of the next slab is issued one slab-time before it is needed, less than the L2 latency).
template <int KG, int GKT>
static __global__ void __launch_bounds__(128 * KG)
gemm_nt_kernel(const GemmDesc *descs, const GemmTile *tiles, const double *baseA, const double *baseB,
               double *baseC, const int *gatherBase) {
  const GemmTile tl = tiles[blockIdx.x];
  const GemmDesc g = descs[tl.prob];
  const double *gA = baseA + g.offA, *gB = baseB + g.offB;
  double *gC = baseC + g.offC;
  const int *gather = (g.gatherOff >= 0) ? gatherBase + g.gatherOff : nullptr;
  const int i0 = tl.ti * GT, c0 = tl.tj * GT;
  extern __shared__ __align__(16) double gemm_sm[];
  double (*As)[GKT][GT + 4] = (double (*)[GKT][GT + 4])gemm_sm;                       // [GST][GKT][GT+4]
  double (*Bs)[GKT][GT + 4] = (double (*)[GKT][GT + 4])(gemm_sm + GST * GKT * (GT + 4));
  // k-range that can be nonzero for this tile
  int klo = 0, khi = g.K;
  if (g.a_tri == TRI_K_LE_ROW) khi = min(khi, i0 + GT);
  if (g.a_tri == TRI_K_GE_ROW) klo = max(klo, i0);
  if (g.b_tri == TRI_K_LE_ROW) khi = min(khi, c0 + GT);
  if (g.b_tri == TRI_K_GE_ROW) klo = max(klo, c0);
  klo = (klo / GKT) * GKT;
  const bool vecA = ((((unsigned long long)gA) & 15) == 0) && ((g.lda & 1) == 0);
  const bool vecB = ((((unsigned long long)gB) & 15) == 0) && ((g.ldb & 1) == 0);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int wr = (warp & 1) * 32, wc = ((warp >> 1) & 1) * 32, kgrp = warp >> 2;
  const int qr = lane >> 2, qc = lane & 3;        // fragment coordinates
  double acc[4][4][2];
#pragma unroll
  for (int a = 0; a < 4; a++)
#pragma unroll
    for (int b = 0; b < 4; b++) { acc[a][b][0] = 0.0; acc[a][b][1] = 0.0; }
  // fragments of this warp's 32x32 sub-tile that hold entries of C (a 200 x 200 block covers 25 x 25 of the 32 x 32
  // fragments its four 64-tiles span: computing all of them cost 1.64 x the DMMAs)
  int variant = -1;
  {
    const int nra = max(0, min(4, (g.M - (i0 + wr) + 7) >> 3)), ncb = max(0, min(4, (g.N - (c0 + wc) + 7) >> 3));
    if (nra > 0 && ncb > 0 && !(g.lower && i0 + wr + 31 < c0 + wc))
      variant = (g.lower && i0 + wr == c0 + wc && nra == ncb) ? 16 + nra - 1 : (nra - 1) * 4 + (ncb - 1);
  }
  const int nslab = khi > klo ? (khi - klo + GKT - 1) / GKT : 0;
  // prologue: GST-1 slabs in flight (a group is committed per slot even when empty, so the wait counts stay uniform)
#pragma unroll
  for (int s = 0; s < GST - 1; s++) {
    if (s < nslab) {
      gemm_stage_slab<KG, GKT>(As[s], gA, g.lda, g.M, i0, g.K, klo + s * GKT, g.a_tri, gather, vecA);
      gemm_stage_slab<KG, GKT>(Bs[s], gB, g.ldb, g.N, c0, g.K, klo + s * GKT, g.b_tri, nullptr, vecB);
    }
    cp_async_commit();
  }
  for (int s = 0; s < nslab; s++) {
    const int buf = s % GST;
    cp_async_wait_group<GST - 2>();                // slab s has landed
    __syncthreads();                               // ... for everyone; and everyone is done with slab s-1
    {
      const int sn = s + GST - 1;                  // refill the buffer slab s-1 just released
      if (sn < nslab) {
        const int k0 = klo + sn * GKT;
        gemm_stage_slab<KG, GKT>(As[sn % GST], gA, g.lda, g.M, i0, g.K, k0, g.a_tri, gather, vecA);
        gemm_stage_slab<KG, GKT>(Bs[sn % GST], gB, g.ldb, g.N, c0, g.K, k0, g.b_tri, nullptr, vecB);
      }
      cp_async_commit();
    }
    gemm_warp_mma<KG, GKT>(acc, As[buf], Bs[buf], wr, wc, qr, qc, kgrp, variant);
  }
  // add the two k-groups: group 1 parks its partial tile in the (now idle) staging buffers
  cp_async_wait_all();
  if (KG == 2) {
    __syncthreads();
    double *red = &As[0][0][0];                      // 2*GKT*(GT+4) doubles >= 4 warps x 32 lanes x 16 values
    const int slot = (warp & 3) * 32 + lane;          // value v of thread t lives at [v*128 + t]: conflict-free
    if (kgrp == 1) {
#pragma unroll
      for (int a = 0; a < 4; a++)
#pragma unroll
        for (int b = 0; b < 4; b++) { red[(a * 4 + b) * 128 + slot] = acc[a][b][0]; }
    }
    __syncthreads();
    if (kgrp == 0) {
#pragma unroll
      for (int a = 0; a < 4; a++)
#pragma unroll
        for (int b = 0; b < 4; b++) acc[a][b][0] += red[(a * 4 + b) * 128 + slot];
    }
    __syncthreads();
    double *red2 = &Bs[0][0][0];
    if (kgrp == 1) {
#pragma unroll
      for (int a = 0; a < 4; a++)
#pragma unroll
        for (int b = 0; b < 4; b++) { red2[(a * 4 + b) * 128 + slot] = acc[a][b][1]; }
    }
    __syncthreads();
    if (kgrp == 0) {
#pragma unroll
      for (int a = 0; a < 4; a++)
#pragma unroll
        for (int b = 0; b < 4; b++) acc[a][b][1] += red2[(a * 4 + b) * 128 + slot];
    }
  }
  if (kgrp != 0) return;
  // C fragment: row = lane/4, cols = 2*(lane%4) + {0,1}
#pragma unroll
  for (int a = 0; a < 4; a++)
#pragma unroll
    for (int b = 0; b < 4; b++)
#pragma unroll
      for (int e = 0; e < 2; e++) {
        int gi = i0 + wr + 8 * a + qr, gc = c0 + wc + 8 * b + 2 * qc + e;
        if (gi < g.M && gc < g.N && (!g.lower || gi >= gc)) {
          double *p = gC + gi + (long long)gc * g.ldc;
          double v = g.alpha * acc[a][b][e];
          *p = g.accumulate ? (*p + v) : v;
        }
      }
}

// Launch: one CTA per tile.  With tiles to spare: 128 threads, no k-split (more CTAs per SM).  With few tiles: the
// k-split variant; with less than two waves of tiles (small batches, e.g. one rank's share of a sharded problem) the
// k-split variant with 32-deep slabs -- a launch is then a chain of slab hand-overs (wait, barrier, refill), and
// halving their number matters more than occupancy (3 x 2 x 32 x 68 doubles = 102 KB per CTA).
static const int GEMM_SMEM_DEEP = GST * 2 * 32 * (GT + 4) * 8;
static inline void gemm_nt_launch(int ntiles, int sm_count, cudaStream_t st, const GemmDesc *descs, const GemmTile *tiles,
                                  const double *baseA, const double *baseB, double *baseC, const int *gatherBase) {
  if (ntiles <= 0) return;
  static bool attr_done = false;
  if (!attr_done) {
    cudaFuncSetAttribute(gemm_nt_kernel<1, GK>, cudaFuncAttributeMaxDynamicSharedMemorySize, GEMM_SMEM);
    cudaFuncSetAttribute(gemm_nt_kernel<2, GK>, cudaFuncAttributeMaxDynamicSharedMemorySize, GEMM_SMEM);
    cudaFuncSetAttribute(gemm_nt_kernel<2, 32>, cudaFuncAttributeMaxDynamicSharedMemorySize, GEMM_SMEM_DEEP);
    attr_done = true;
  }
  if (ntiles >= 6 * sm_count) gemm_nt_kernel<1, GK><<<ntiles, 128, GEMM_SMEM, st>>>(descs, tiles, baseA, baseB, baseC, gatherBase);
  else if (ntiles >= 2 * sm_count) gemm_nt_kernel<2, GK><<<ntiles, 256, GEMM_SMEM, st>>>(descs, tiles, baseA, baseB, baseC, gatherBase);
  else gemm_nt_kernel<2, 32><<<ntiles, 256, GEMM_SMEM_DEEP, st>>>(descs, tiles, baseA, baseB, baseC, gatherBase);
}

// Host helper: append the tiles of one problem to a tile list.
template <typename Vec>
inline void gemm_add_tiles(Vec &tiles, int prob, int M, int N, bool lower) {
  for (int tj = 0; tj * GT < N; tj++)
    for (int ti = 0; ti * GT < M; ti++) {
      if (lower && (ti + 1) * GT - 1 < tj * GT) continue;
      tiles.push_back(GemmTile{prob, ti, tj});
    }
}

}  // namespace sb
