// ada_fused.cuh -- getada3 for PSD blocks up to order 208: W_jk never leaves the SM.
//
// One CTA works on one (constraint j, PSD block k) pair at a time (pairs are handed out by an atomic counter):
//   1. T = sym(A_jk)(R,:) D_k, r x n, written to this CTA's private scratch slot (global memory, but the slot is
//      re-used for every pair the CTA processes, so it lives in L2 and is never streamed from HBM);
//   2. W = D_k(:,R) T on the FP64 tensor pipe (DMMA m8n8k4): a warp owns one 32x32 supertile of the LOWER triangle
//      per round (4x4 fragments, clipped at the diagonal and at n; n = 200 needs two rounds of 16 warps), operands
//      staged through a two-stage cp.async ring of 8-deep k-slabs; the accumulators go to shared memory as the
//      packed lower triangle of W;
//   3. every constraint i of block k that precedes j in the ordering takes <A_ik, W> from shared memory
//      (dots_partners, the same code the unfused kernel uses), writes ADA(i,j) / per-pair partial sums and absd.
// The unfused path materialised W (n^2 doubles per pair) in HBM between a GEMM launch and a dots launch: several
// times the algorithmic traffic of getada3.  Reference: getada3.c:305-351, spscale.c:249-305.
#pragma once

namespace sb {

static const int FUSED_MAX_N = 208;                 // 7 x 7 supertiles -> 28 warps; W (packed) + the staging ring fit 227 KB
static const int FKC = 8;                            // k-slab depth (two DMMA k-steps)
static const int FUSED_GEMM_WARPS = 16;              // warps that hold a 32x32 accumulator tile in one round
static const int FTK = 8, FTST = 2;                  // TMA ring: k-depth of a slab, stages (FTK * FTST == 2 * FKC: same shared memory;
                                                     // 4 x 4 is slower: twice the barrier hand-overs per DMMA)

struct FusedArgs {
  const AdaPair *pairs; int npairs;
  int *counter;
  const int *blk_n; const long long *blk_off;
  const int *tt_ptr, *tt_col, *tt_row; const double *tt_val;  // per (pair, row of R): entries (column, row, weight*value)
  const int *Rlist;
  const double *udsqr;
  double *scratch; long long scratch_stride;         // per-CTA T slot
  // dots
  const long long *adajc; const int *adair; const int *invperm; int first;
  const int *cpair_beg; const int *blkp_beg; const BlkPartner *blkp;
  const int *ent_pk; const int *ent_src; const double *Atpr;
  double *ws, *ada, *absd;
  const int *blk_group;
  const int *blk_item_beg; const int2 *items;        // per block: its lower supertiles (I, J), most expensive first
  const int *need_pq; const int *order;              // entry-wise pairs: their (p | q << 16) lists; processing order of the pairs
  int wcap, ldmax;
  const int *slot;                                   // per pair: ADA positions of its partners (AdaPair::slot_off)
  unsigned long long *prof;                          // optional: cycles per phase summed over CTAs (thread 0's clock), 8 slots
};

__device__ __forceinline__ int fused_ld(int n) { return ((n + 7) & ~7) + 4; }   // == 4 (mod 8): conflict-free fragment loads

// one k-slab of both operands, global -> shared:  As[kk][p] = D[p + R[k0+kk] n],  Bs[kk][q] = Tt[q + (k0+kk) n].
// Thread t serves k-row kk = t / TPR with TPR = blockDim / 8 threads per row (no divisions: TPR is a power of two).
template <int TPR_LOG2>
__device__ __forceinline__ void fused_stage(double *As, double *Bs, int ld, const double *D, const double *Tt, const int *R,
                                            int n, int r, int k0, bool vec) {
  const int kk = threadIdx.x >> TPR_LOG2, l = threadIdx.x & ((1 << TPR_LOG2) - 1), k = k0 + kk;
  const unsigned sa = (unsigned)__cvta_generic_to_shared(As + kk * ld), sb = (unsigned)__cvta_generic_to_shared(Bs + kk * ld);
  if (k < r) {
    const double *srcA = D + (long long)R[k] * n, *srcB = Tt + (long long)k * n;
    if (vec) {                                       // n even, 16-byte aligned bases
      for (int p = 2 * l; p < n; p += 2 << TPR_LOG2) {
        asm volatile("cp.async.cg.shared.global [%0], [%1], 16;\n" :: "r"(sa + 8u * p), "l"(srcA + p) : "memory");
        asm volatile("cp.async.cg.shared.global [%0], [%1], 16;\n" :: "r"(sb + 8u * p), "l"(srcB + p) : "memory");
      }
    } else {
      for (int p = l; p < n; p += 1 << TPR_LOG2) {
        asm volatile("cp.async.ca.shared.global [%0], [%1], 8;\n" :: "r"(sa + 8u * p), "l"(srcA + p) : "memory");
        asm volatile("cp.async.ca.shared.global [%0], [%1], 8;\n" :: "r"(sb + 8u * p), "l"(srcB + p) : "memory");
      }
    }
  } else {                                           // beyond K: zero rows
    for (int p = l; p < n; p += 1 << TPR_LOG2) { As[kk * ld + p] = 0.0; Bs[kk * ld + p] = 0.0; }
  }
}

// ---- mbarrier / TMA (1-D bulk copy) helpers of the operand ring
__device__ __forceinline__ unsigned f_smem_u32(const void *p) { return (unsigned)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void f_mbar_init(unsigned bar, unsigned count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;\n" :: "r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void f_mbar_expect_tx(unsigned bar, unsigned bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;\n" :: "r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void f_mbar_arrive(unsigned bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];\n" :: "r"(bar) : "memory");
}
__device__ __forceinline__ void f_mbar_wait(unsigned bar, unsigned parity) {
  asm volatile("{\n .reg .pred P1;\n LAB_WAIT:\n mbarrier.try_wait.parity.shared::cta.b64 P1, [%0], %1;\n @P1 bra DONE;\n bra LAB_WAIT;\n DONE:\n }\n"
               :: "r"(bar), "r"(parity) : "memory");
}
__device__ __forceinline__ void f_bulk_g2s(unsigned dst, const void *src, unsigned bytes, unsigned bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];\n"
               :: "r"(dst), "l"(src), "r"(bytes), "r"(bar) : "memory");
}

// The DMMAs of one k-slab on a warp's supertile.  The supertile shapes that occur are known when the plan is built:
// interior (4 x 4 fragments), diagonal (lower triangle of NRA x NRA) and row-clipped (NRA x 4, the last supertile row);
// each gets straight-line code.  (A run-time fragment mask compiled to one predicated DMMA + WARPSYNC per fragment slot:
// the second round of n = 200 -- a quarter of the first round's DMMAs -- took 30 % longer than the first.)
template <int NRA, bool DIAG, int KD>
__device__ __forceinline__ void fused_slab_mma_static(double (&acc)[4][4][2], const double *As, const double *Bs, int ld, int qc) {
  constexpr int NCB = DIAG ? NRA : 4;
#pragma unroll
  for (int k4 = 0; k4 < KD; k4 += 4) {
    double af[4], bf[4];
#pragma unroll
    for (int a = 0; a < NRA; a++) af[a] = As[(k4 + qc) * ld + 8 * a];
#pragma unroll
    for (int b = 0; b < NCB; b++) bf[b] = Bs[(k4 + qc) * ld + 8 * b];
#pragma unroll
    for (int a = 0; a < NRA; a++)
#pragma unroll
      for (int b = 0; b < NCB; b++)
        if (!DIAG || a >= b) dmma_m8n8k4(acc[a][b][0], acc[a][b][1], af[a], bf[b]);
  }
}
// variant = NRA - 1 (row-clipped or interior), 4 + NRA - 1 (diagonal), -1: nothing to do
template <int KD>
__device__ __forceinline__ void fused_slab_mma(double (&acc)[4][4][2], const double *As, const double *Bs, int ld, int qc, int variant) {
  switch (variant) {
    case 3: fused_slab_mma_static<4, false, KD>(acc, As, Bs, ld, qc); break;
    case 7: fused_slab_mma_static<4, true, KD>(acc, As, Bs, ld, qc); break;
    case 0: fused_slab_mma_static<1, false, KD>(acc, As, Bs, ld, qc); break;
    case 1: fused_slab_mma_static<2, false, KD>(acc, As, Bs, ld, qc); break;
    case 2: fused_slab_mma_static<3, false, KD>(acc, As, Bs, ld, qc); break;
    case 4: fused_slab_mma_static<1, true, KD>(acc, As, Bs, ld, qc); break;
    case 5: fused_slab_mma_static<2, true, KD>(acc, As, Bs, ld, qc); break;
    case 6: fused_slab_mma_static<3, true, KD>(acc, As, Bs, ld, qc); break;
    default: break;
  }
}

template <int NTHREADS, int MINB>
__global__ void __launch_bounds__(NTHREADS, MINB) ada3_fused_kernel(const FusedArgs A) {
  extern __shared__ __align__(16) double fsm[];
  double *Wp = fsm;                                             // packed lower triangle of W, wcap doubles
  double *stA = fsm + A.wcap;                                   // [2][FKC][ldmax]
  double *stB = stA + 2 * FKC * A.ldmax;
  __shared__ int s_pair[2];
  __shared__ int sR[FUSED_MAX_N], sPtr[FUSED_MAX_N + 1];       // the pair's row list and row pointers (staging and the T
                                                                // loop would otherwise start every step with a global load)
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, nw = blockDim.x >> 5;
  const int qr = lane >> 2, qc = lane & 3;
  double *Tt = A.scratch + (long long)blockIdx.x * A.scratch_stride;
  // operand ring of the dense products: FTST stages of FTK k-values, each filled by 2 FTK TMA bulk copies (columns of D, rows of T)
  // that complete on the stage's `full` mbarrier; a stage is handed back through its `empty` mbarrier (one arrival per
  // warp).  No block-wide barrier inside the k loop: a warp only waits for data, the producer only for a free stage.
  __shared__ __align__(8) unsigned long long s_full[FTST], s_empty[FTST];
  if (tid == 0) {
    s_pair[0] = atomicAdd(A.counter, 1);
    for (int i = 0; i < FTST; i++) { f_mbar_init(f_smem_u32(&s_full[i]), 1); f_mbar_init(f_smem_u32(&s_empty[i]), nw); }
    asm volatile("fence.mbarrier_init.release.cluster;\n" ::: "memory");
  }
  __syncthreads();
  unsigned gslab = 0;                                           // slabs that went through the ring so far (same in every thread)
#ifdef SB200_FUSED_PROF
  long long pc[14] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0};         // cycles per phase (thread 0), see sb200_ada_fused_profile
#define FPROF(...) __VA_ARGS__
#else
#define FPROF(...)
#endif
  for (int turn = 0;; turn ^= 1) {
    const int cur = s_pair[turn];
    if (cur >= A.npairs) break;
    FPROF(long long c0k = clock64();)
    int nxt = 0;
    if (tid == 0) nxt = atomicAdd(A.counter, 1);               // the next pair's ticket travels while this one is worked on
    const int pi = A.order[cur];
    const AdaPair P = A.pairs[pi];
    const int n = A.blk_n[P.k], r = P.r, ld = fused_ld(n);
    const double *D = A.udsqr + A.blk_off[P.k];
    const int *R = sR;
    const int r8 = (r + FKC - 1) & ~(FKC - 1);                  // the ring moves whole slabs: rows r..r8 of T are zero,
    for (int i = tid; i < r8; i += blockDim.x) sR[i] = A.Rlist[P.r0 + (i < r ? i : 0)];     // paired with any valid column of D
    for (int i = tid; i <= r; i += blockDim.x) sPtr[i] = A.tt_ptr[P.r0 + i];
    __syncthreads();
    FPROF(if (tid == 0) { const long long c = clock64(); pc[0] += c - c0k; c0k = c; })
    // ---------------- 1. T (as Tt: n x r, column rho = row R[rho] of sym(A) D): one warp per row, lanes over columns
    if (P.mode != 2) {
      const int *ptr = sPtr;
      const bool vec2 = ((n & 1) == 0) && ((((unsigned long long)D) & 15) == 0) && ((((unsigned long long)Tt) & 15) == 0);
      if (vec2) {                                                // two columns per lane and load
        constexpr int NCH = (FUSED_MAX_N / 2 + 31) / 32;
        const int half = n >> 1;
        // the warp walks its rows as ONE stream of 4-entry trips; the (column, value) of the next trip -- of this row
        // or of the warp's next row -- are fetched before the loads of D of the current trip are consumed, so a trip
        // exposes one L2 round trip instead of two
        int rho = warp;
        int t = rho < r ? ptr[rho] : 0, te = rho < r ? ptr[rho + 1] : 0;
        int col[4]; double v[4];
#pragma unroll
        for (int u = 0; u < 4; u++) {
          const bool ok = t + u < te;
          v[u] = ok ? A.tt_val[t + u] : 0.0;
          col[u] = ok ? A.tt_col[t + u] : 0;
        }
        double2 acc[NCH];
#pragma unroll
        for (int ch = 0; ch < NCH; ch++) acc[ch] = make_double2(0.0, 0.0);
        while (rho < r) {
          int nrho = rho, nt = t + 4, nte = te;
          if (nt >= te) { nrho = rho + nw; nt = nrho < r ? ptr[nrho] : 0; nte = nrho < r ? ptr[nrho + 1] : 0; }
          int ncol[4]; double nv[4];
#pragma unroll
          for (int u = 0; u < 4; u++) {
            const bool ok = nt + u < nte;
            nv[u] = ok ? A.tt_val[nt + u] : 0.0;
            ncol[u] = ok ? A.tt_col[nt + u] : 0;
          }
          const double2 *Dc0 = reinterpret_cast<const double2 *>(D + (long long)col[0] * n);
          const double2 *Dc1 = reinterpret_cast<const double2 *>(D + (long long)col[1] * n);
          const double2 *Dc2 = reinterpret_cast<const double2 *>(D + (long long)col[2] * n);
          const double2 *Dc3 = reinterpret_cast<const double2 *>(D + (long long)col[3] * n);
#pragma unroll
          for (int ch = 0; ch < NCH; ch++) {
            const int c = lane + 32 * ch;
            if (c < half) {
              const double2 x0 = Dc0[c], x1 = Dc1[c], x2 = Dc2[c], x3 = Dc3[c];
              acc[ch].x += v[0] * x0.x; acc[ch].y += v[0] * x0.y;
              acc[ch].x += v[1] * x1.x; acc[ch].y += v[1] * x1.y;
              acc[ch].x += v[2] * x2.x; acc[ch].y += v[2] * x2.y;
              acc[ch].x += v[3] * x3.x; acc[ch].y += v[3] * x3.y;
            }
          }
          if (nrho != rho) {
            double2 *dst = reinterpret_cast<double2 *>(Tt + (long long)rho * n);
#pragma unroll
            for (int ch = 0; ch < NCH; ch++) {
              const int c = lane + 32 * ch;
              if (c < half) dst[c] = acc[ch];
              acc[ch] = make_double2(0.0, 0.0);
            }
          }
          rho = nrho; t = nt; te = nte;
#pragma unroll
          for (int u = 0; u < 4; u++) { col[u] = ncol[u]; v[u] = nv[u]; }
        }
      } else {
        constexpr int NCH = (FUSED_MAX_N + 31) / 32;
        for (int rho = warp; rho < r; rho += nw) {
          double acc[NCH];
#pragma unroll
          for (int ch = 0; ch < NCH; ch++) acc[ch] = 0.0;
          const int t0 = ptr[rho], t1 = ptr[rho + 1];
          for (int t = t0; t < t1; t++) {
            const double v = A.tt_val[t];
            const double *Dc = D + (long long)A.tt_col[t] * n;
#pragma unroll
            for (int ch = 0; ch < NCH; ch++) {
              const int c = lane + 32 * ch;
              if (c < n) acc[ch] += v * Dc[c];
            }
          }
          double *dst = Tt + (long long)rho * n;
#pragma unroll
          for (int ch = 0; ch < NCH; ch++) {
            const int c = lane + 32 * ch;
            if (c < n) dst[c] = acc[ch];
          }
        }
      }
    }
    if (P.mode == 0) {
      for (int rho = r + warp; rho < r8; rho += nw)
        for (int c = lane; c < n; c += 32) Tt[(long long)rho * n + c] = 0.0;
      asm volatile("fence.proxy.async;\n" ::: "memory");       // T was written through the generic proxy, TMA reads it
    }
    __syncthreads();
    FPROF(if (tid == 0) { const long long c = clock64(); pc[1] += c - c0k; c0k = c; })
    // ---------------- 2a. entry-wise evaluation on the needed set (pairs early in their block's list)
    if (P.mode != 0) {
      // four lanes share one needed entry (p, q) and split the sum; eight terms per lane are in flight at a time
      const int *pq = A.need_pq + P.need_off;
      const int g = tid & 3;
      const int e0 = sPtr[0], e1 = sPtr[r];
      // mode 2: the pair's (value, row, column) list -- at most 2 n entries -- moves into the idle operand ring once, so a
      // term of the sums below costs the two loads of D and nothing else from global memory
      double *sval = stA;
      int *srow = reinterpret_cast<int *>(stA + 2 * FUSED_MAX_N), *scol = srow + 2 * FUSED_MAX_N;
      const int cnt = e1 - e0;
      const bool staged = P.mode == 2 && cnt <= 2 * FUSED_MAX_N && 2 * FUSED_MAX_N * 2 <= 2 * FKC * A.ldmax;
      if (staged) {
        for (int t = tid; t < cnt; t += blockDim.x) { sval[t] = A.tt_val[e0 + t]; srow[t] = A.tt_row[e0 + t]; scol[t] = A.tt_col[e0 + t]; }
        __syncthreads();
      }
      for (int u0 = 0; u0 < P.need_cnt; u0 += (int)(blockDim.x >> 2)) {
        const int u = u0 + (tid >> 2);
        const bool live = u < P.need_cnt;
        const int v = live ? pq[u] : 0, pp = v & 0xffff, qq = v >> 16;
        double acc = 0.0;
        if (P.mode == 1) {                                        // through T: sum_rho D(p,R[rho]) T(rho,q)
          if (live) {
#pragma unroll 8
            for (int rho = g; rho < r; rho += 4) acc += D[pp + (long long)R[rho] * n] * Tt[qq + (long long)rho * n];
          }
        } else {                                                  // few entries in A_jk: sum_t v_t D(p,row_t) D(col_t,q), D symmetric
          if (live && staged) {
#pragma unroll 8
            for (int t = g; t < cnt; t += 4) {
              const int a1 = pp + srow[t] * n, a2 = qq + scol[t] * n;
              const double d1 = D[a1];
              const double d2 = a2 == a1 ? d1 : D[a2];            // diagonal entry of W from a diagonal entry of A: one load
              acc += sval[t] * (d1 * d2);
            }
          } else if (live) {
#pragma unroll 8
            for (int t = e0 + g; t < e1; t += 4)
              acc += A.tt_val[t] * (D[pp + (long long)A.tt_row[t] * n] * D[qq + (long long)A.tt_col[t] * n]);
          }
        }
        acc += __shfl_xor_sync(0xffffffffu, acc, 1);
        acc += __shfl_xor_sync(0xffffffffu, acc, 2);
        if (live && g == 0) Wp[(qq * (2 * n - qq + 1)) / 2 - qq + pp] = acc;
      }
      if (staged) asm volatile("fence.proxy.async;\n" ::: "memory");   // the ring is written by TMA again for the next dense pair
    } else
    // ---------------- 2b. W = D(:,R) T on the lower supertiles, in rounds of at most FUSED_GEMM_WARPS items
    // (the accumulators of the whole lower triangle -- 325 fragments at n = 200 -- do not fit the register file next to
    // anything else; the planner sorts the items of a block by cost, so a round costs what its first item costs)
    {
      const int ib = A.blk_item_beg[P.k], ie = A.blk_item_beg[P.k + 1];
      const int nwg = min(nw, FUSED_GEMM_WARPS);
      const bool vec = ((n & 1) == 0) && ((((unsigned long long)D) & 15) == 0) && ((((unsigned long long)Tt) & 15) == 0);
      const int nslab = (r + FKC - 1) / FKC;
      for (int it0 = ib; it0 < ie; it0 += nwg) {
        const bool have = warp < nwg && it0 + warp < ie;
        const int2 IJ = have ? A.items[it0 + warp] : make_int2(0, 0);
        const int rb = 32 * IJ.x, cb = 32 * IJ.y;
        const int nra = have ? min(4, (n - rb + 7) >> 3) : 0;       // fragment rows / columns inside n
        const int ncb = have ? min(4, (n - cb + 7) >> 3) : 0;
        const bool diag = (IJ.x == IJ.y);
        // a non-diagonal supertile of the lower triangle lies strictly left of the last supertile column: ncb == 4
        const int variant = have ? (diag ? 4 : 0) + nra - 1 : -1;
        double acc[4][4][2];
#pragma unroll
        for (int a = 0; a < 4; a++)
#pragma unroll
          for (int b = 0; b < 4; b++) { acc[a][b][0] = 0.0; acc[a][b][1] = 0.0; }
        if (vec) {
          // ---- TMA ring
          const unsigned row_bytes = 8u * (unsigned)n;
          const int nslab8 = r8 / FTK;
          // the producer is the LAST warp: the planner sorts a round's supertiles by cost, so it holds the cheapest one
          // (or none) and its wait for a free stage is off the critical path.  FTST - 1 slabs are in flight ahead of the
          // one being consumed: a round of cheap supertiles is bound by the copy rate, not by one L2 latency per slab.
          auto issue = [&](int sl) {                              // slab sl of this round (producer warp only)
            const unsigned gs = gslab + (unsigned)sl, st = gs % FTST, use = gs / FTST;
            if (use > 0) f_mbar_wait(f_smem_u32(&s_empty[st]), (use - 1u) & 1u);      // every warp is done with the stage
            if (lane == 0) f_mbar_expect_tx(f_smem_u32(&s_full[st]), 2u * FTK * row_bytes);
            __syncwarp();
            if (lane < 2 * FTK) {
              const int kk = lane & (FTK - 1), k = sl * FTK + kk;
              const double *src = lane < FTK ? D + (long long)sR[k] * n : Tt + (long long)k * n;
              double *dst = (lane < FTK ? stA : stB) + (st * FTK + kk) * A.ldmax;
              f_bulk_g2s(f_smem_u32(dst), src, row_bytes, f_smem_u32(&s_full[st]));
            }
          };
          if (warp == nw - 1)
            for (int sl = 0; sl < FTST - 1 && sl < nslab8; sl++) issue(sl);
          for (int sl = 0; sl < nslab8; sl++) {
            FPROF(long long q0 = clock64();)
            if (warp == nw - 1 && sl + FTST - 1 < nslab8) issue(sl + FTST - 1);
            FPROF(if (tid == 0) { const long long c = clock64(); pc[it0 == ib ? 8 : 12] += c - q0; q0 = c; })
            const unsigned gs = gslab + (unsigned)sl, st = gs % FTST, use = gs / FTST;
            f_mbar_wait(f_smem_u32(&s_full[st]), use & 1u);
            FPROF(if (tid == 0) { const long long c = clock64(); pc[it0 == ib ? 7 : 11] += c - q0; q0 = c; })
            const double *As = stA + st * FTK * A.ldmax + rb + qr, *Bs = stB + st * FTK * A.ldmax + cb + qr;
            fused_slab_mma<FTK>(acc, As, Bs, A.ldmax, qc, variant);
            __syncwarp();
            if (lane == 0) f_mbar_arrive(f_smem_u32(&s_empty[st]));
            FPROF(if (tid == 0) { const long long c = clock64(); pc[it0 == ib ? 9 : 13] += c - q0; })
          }
          gslab += (unsigned)nslab8;
        } else {
        constexpr int TPR_LOG2 = (NTHREADS == 512) ? 6 : 5;       // 8 k-rows x TPR threads = blockDim
        if (nslab > 0) fused_stage<TPR_LOG2>(stA, stB, ld, D, Tt, R, n, r, 0, vec);
        cp_async_commit();
        for (int s = 0; s < nslab; s++) {
          const int buf = s & 1;
          cp_async_wait_all();
          __syncthreads();                                        // slab s visible; everyone is done with slab s-1
          if (s + 1 < nslab) fused_stage<TPR_LOG2>(stA + (buf ^ 1) * FKC * A.ldmax, stB + (buf ^ 1) * FKC * A.ldmax, ld, D, Tt, R, n, r, (s + 1) * FKC, vec);
          cp_async_commit();
          const double *As = stA + buf * FKC * A.ldmax + rb + qr, *Bs = stB + buf * FKC * A.ldmax + cb + qr;
          fused_slab_mma<FKC>(acc, As, Bs, ld, qc, variant);
        }
        }
        FPROF(long long q1 = clock64();)
        cp_async_wait_all();
        // accumulators -> packed lower triangle: (p, q), p >= q, at q (2n - q + 1)/2 - q + p
#pragma unroll
        for (int a = 0; a < 4; a++)
#pragma unroll
          for (int b = 0; b < 4; b++)
#pragma unroll
            for (int e = 0; e < 2; e++) {
              const int p = rb + 8 * a + qr, q = cb + 8 * b + 2 * qc + e;
              if (a < nra && b < ncb && p < n && q < n && p >= q) Wp[(q * (2 * n - q + 1)) / 2 - q + p] = acc[a][b][e];
            }
        __syncthreads();                                          // the ring is re-used by the next round
        FPROF(if (tid == 0) pc[10] += clock64() - q1;)
      }
    }
    __syncthreads();
    FPROF(if (tid == 0) { const long long c = clock64(); pc[P.mode == 0 ? 2 : 3] += c - c0k; c0k = c; if (P.mode == 0) pc[5]++; else pc[6]++; })
    // ---------------- 3. inner products with the partners of block k
    {
      const int c = P.j;
      const bool multi = A.cpair_beg[c + 1] - A.cpair_beg[c] > 1;
      const int ipc = A.invperm[c];
      const long long colbeg = A.adajc[c];
      ColSlots cs{A.adair + colbeg, (int)(A.adajc[c + 1] - colbeg), nullptr};
      if (!multi) {
        if (tid == 0) {
          const int sd = ipc >= A.first ? cs.find(c) : -1;
          A.absd[c] = sd >= 0 ? A.ada[colbeg + sd] : 0.0;
        }
        __syncthreads();
      }
      DotsCtx X;
      X.rank_limit = P.rank;
      X.P = P; X.P.part_off = P.fpart_off; X.c = c; X.ipc = ipc; X.first = A.first; X.multi = multi ? 1 : 0;
      X.warp = warp; X.lane = lane; X.nw = nw; X.colbeg = colbeg; X.cs = cs; X.eidx = A.ent_pk; X.Wp = Wp;
      X.blkp_beg = A.blkp_beg; X.blkp = A.blkp; X.invperm = A.invperm; X.Atpr = A.Atpr; X.ent_src = A.ent_src;
      X.ent_scale = nullptr; X.ws = A.ws; X.ada = A.ada; X.absd = A.absd; X.slot_tab = A.slot + P.slot_off;
      switch (A.blk_group[P.k]) {
        case 4: dots_partners<4>(X); break;
        case 8: dots_partners<8>(X); break;
        case 16: dots_partners<16>(X); break;
        default: dots_partners<32>(X); break;
      }
    }
    if (tid == 0) s_pair[turn ^ 1] = nxt;
    __syncthreads();                                            // Wp, sR / sPtr and the scratch slot are re-used by the next pair
    FPROF(if (tid == 0) { const long long c = clock64(); pc[4] += c - c0k; })
  }
  FPROF(if (tid == 0 && A.prof) for (int i = 0; i < 14; i++) atomicAdd(A.prof + i, (unsigned long long)pc[i]);)
}

}  // namespace sb
