// ada_strip.cuh -- getada3 for PSD blocks whose packed W does not leave room for a second resident CTA (orders 97..208).
//
// ada_fused.cuh keeps the whole packed lower triangle of W_jk in shared memory (160 KB at n = 200): one CTA per SM, and
// its phases -- T = sym(A_jk) D (L2 latency), W = D T (FP64 tensor pipe), <A_ik, W> (L2 latency + shared memory) -- run
// one after the other with nothing to overlap them (the DMMA pipe idles outside the product phase).  Here the unit of work is a (pair, column strip) instead of a pair:
//   * the lower triangle is cut into strips of whole supertile columns (<= STRIP_WCAP entries, <= 8 supertiles: one
//     round of 8 warps); a strip is a CONTIGUOUS range of the packed index, so W_strip is a plain sub-array;
//   * only the strip's columns of T are built (the strips of a pair partition T: no work is duplicated) and only rows
//     >= c0 of D(:,R) are staged;
//   * every partner's entries are pre-sorted by strip (16-bit index relative to the strip + value, 10 bytes per entry
//     instead of 12), its partial inner product goes to a per-(pair, strip) slot, and ada3_strip_reduce_kernel adds
//     the strips of a pair in a fixed order (deterministic, no atomics on ADA).
// 90 KB of shared memory and 256 threads per CTA: two CTAs per SM, whose phases interleave.
// Reference: getada3.c:305-351, spscale.c:249-305.
#pragma once

namespace sb {

static const int STRIP_WCAP = 6016;                  // doubles of W per strip
static const int STRIP_THREADS = 256;
static const int STRIP_STAGES = 3;

struct StripGroup { int c0, c1, base, item_beg, item_end, gw_al; };   // columns [c0,c1); packed index of (c0,c0); supertiles; Tt row stride
struct StripPG { long long part_off; int need_beg, need_cnt; };        // per (pair, strip): partial sums (rank+2), needed entries
struct StripWork { int pair, g; };

struct StripArgs {
  const AdaPair *pairs; const StripWork *work; int nwork; int *counter;
  const int *blk_n; const long long *blk_off;
  const int *blk_grp_beg; const StripGroup *groups; const int2 *items;
  const int *pair_pg; const StripPG *pg;
  const int *tt_ptr, *tt_col, *tt_row; const double *tt_val; const int *Rlist; const double *udsqr;
  double *scratch; long long scratch_stride;
  const int *blk_feoff; const int *fe_ptr; const unsigned short *fe_pk; const double *fe_val;
  const int *need_pq;
  double *ws;
  const int *blk_lanes;
  int ldA, ldB;
};

// one k-slab of both operands: As[kk][p - a0] = D[p + R[k0+kk] n] (p >= a0), Bs[kk][q - c0] = Tt[(q - c0) + (k0+kk) gwa]
__device__ __forceinline__ void strip_stage(double *As, double *Bs, int ldA, int ldB, const double *D, const double *Tt, const int *R,
                                            int n, int r, int k0, int a0, int gw, int gwa, bool vec) {
  const int kk = threadIdx.x >> 5, l = threadIdx.x & 31, k = k0 + kk;
  const int na = n - a0;
  const unsigned sa = (unsigned)__cvta_generic_to_shared(As + kk * ldA), sb = (unsigned)__cvta_generic_to_shared(Bs + kk * ldB);
  if (k < r) {
    const double *srcA = D + (long long)R[k] * n + a0, *srcB = Tt + (long long)k * gwa;
    if (vec) {
      for (int p = 2 * l; p < na; p += 64)
        asm volatile("cp.async.cg.shared.global [%0], [%1], 16;\n" :: "r"(sa + 8u * p), "l"(srcA + p) : "memory");
      for (int q = 2 * l; q < gw; q += 64)
        asm volatile("cp.async.cg.shared.global [%0], [%1], 16;\n" :: "r"(sb + 8u * q), "l"(srcB + q) : "memory");
    } else {
      for (int p = l; p < na; p += 32)
        asm volatile("cp.async.ca.shared.global [%0], [%1], 8;\n" :: "r"(sa + 8u * p), "l"(srcA + p) : "memory");
      for (int q = l; q < gw; q += 32)
        asm volatile("cp.async.ca.shared.global [%0], [%1], 8;\n" :: "r"(sb + 8u * q), "l"(srcB + q) : "memory");
    }
  } else {
    for (int p = l; p < na; p += 32) As[kk * ldA + p] = 0.0;
    for (int q = l; q < gw; q += 32) Bs[kk * ldB + q] = 0.0;
  }
}

// partial inner products of one strip with G lanes per partner
template <int G>
__device__ __forceinline__ void strip_dots(const StripArgs &A, const AdaPair &P, int g, int ng, const double *Wg, double *part,
                                           int warp, int lane, int nw) {
  constexpr int GPW = 32 / G;
  const int grp = lane / G, gl = lane % G;
  const unsigned gmask = G == 32 ? 0xffffffffu : (((1u << G) - 1u) << (grp * G));
  const int *fp = A.fe_ptr + A.blk_feoff[P.k] + g;            // (partner t, strip g) -> fp[t ng], fp[t ng + 1]
  const int tl = P.rank + 1;
  int t = warp * GPW + grp;
  int e0n = 0, e1n = 0;
  if (t < tl) { e0n = fp[(long long)t * ng]; e1n = fp[(long long)t * ng + 1]; }
  for (; t < tl; t += nw * GPW) {
    const int e0 = e0n, e1 = e1n;
    {
      const int tn = t + nw * GPW;
      if (tn < tl) { e0n = fp[(long long)tn * ng]; e1n = fp[(long long)tn * ng + 1]; }
    }
    double acc = 0.0, aabs = 0.0;
    int e = e0 + gl;
    for (; e < e1; e += 8 * G) {                              // 8 entries per lane and trip, 16 loads in flight (see dots_partners)
      double a[8]; int ix[8];
#pragma unroll
      for (int u = 0; u < 8; u++) {
        const bool ok = e + u * G < e1;
        a[u] = ok ? A.fe_val[e + u * G] : 0.0;
        ix[u] = ok ? (int)A.fe_pk[e + u * G] : -1;
      }
#pragma unroll
      for (int u = 0; u < 8; u++) {
        const double term = ix[u] >= 0 ? a[u] * Wg[ix[u]] : 0.0;
        acc += term; aabs += fabs(term);
      }
    }
#pragma unroll
    for (int o = G / 2; o > 0; o >>= 1) {
      acc += __shfl_down_sync(gmask, acc, o, G);
      aabs += __shfl_down_sync(gmask, aabs, o, G);
    }
    if (gl == 0) {
      part[t] = acc;
      if (t == P.rank) part[P.rank + 1] = aabs;             // the pair's own constraint closes its list
    }
  }
}

template <int MINB>
__global__ void __launch_bounds__(STRIP_THREADS, MINB) ada3_strip_kernel(const StripArgs A) {
  extern __shared__ __align__(16) double ssm[];
  double *Wg = ssm;                                             // STRIP_WCAP
  double *stA = ssm + STRIP_WCAP;                               // [STRIP_STAGES][FKC][ldA]
  double *stB = stA + STRIP_STAGES * FKC * A.ldA;               // [STRIP_STAGES][FKC][ldB]
  __shared__ int s_w[2];
  __shared__ int sR[FUSED_MAX_N], sPtr[FUSED_MAX_N + 1];       // the pair's row list and row pointers
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  constexpr int nw = STRIP_THREADS / 32;
  const int qr = lane >> 2, qc = lane & 3;
  double *Tt = A.scratch + (long long)blockIdx.x * A.scratch_stride;
  if (tid == 0) s_w[0] = atomicAdd(A.counter, 1);
  __syncthreads();
  for (int turn = 0;; turn ^= 1) {
    const int cur = s_w[turn];
    if (cur >= A.nwork) break;
    int nxt = 0;
    if (tid == 0) nxt = atomicAdd(A.counter, 1);               // the next ticket travels while this item is worked on
    const StripWork Wk = A.work[cur];
    const AdaPair P = A.pairs[Wk.pair];
    const int n = A.blk_n[P.k], r = P.r;
    const int gb = A.blk_grp_beg[P.k], ng = A.blk_grp_beg[P.k + 1] - gb;
    const StripGroup Gp = A.groups[gb + Wk.g];
    const StripPG PG = A.pg[A.pair_pg[Wk.pair] + Wk.g];
    const int c0 = Gp.c0, gw = Gp.c1 - Gp.c0, gwa = Gp.gw_al;
    const double *D = A.udsqr + A.blk_off[P.k];
    const int *R = sR;
    for (int i = tid; i < r; i += STRIP_THREADS) sR[i] = A.Rlist[P.r0 + i];
    for (int i = tid; i <= r; i += STRIP_THREADS) sPtr[i] = A.tt_ptr[P.r0 + i];
    __syncthreads();
    const bool vec = ((n & 1) == 0) && ((c0 & 1) == 0) && ((gw & 1) == 0) && ((((unsigned long long)D) & 15) == 0) &&
                     ((((unsigned long long)Tt) & 15) == 0);
    // ---------------- 1. the strip's columns of T: Tt[(q - c0) + rho gwa] = sum_t v_t D(q, col_t), q in [c0, c1)
    if (P.mode != 2) {
      // a row of T takes 4 columns per lane: LPR = 8 / 16 / 32 lanes per row, 32 / LPR rows per warp at a time.  Each
      // lane group walks its rows as one stream of 4-entry trips and fetches the (column, value) of the next trip -- of
      // this row or of the group's next row -- before the loads of D of the current trip are consumed: one L2 round
      // trip per trip.  (One row per warp cost 5 x what the whole-pair kernel paid: this loop is pure latency.)
      const int *ptr = sPtr;
      const int lpr_log2 = gw <= 32 ? 3 : (gw <= 64 ? 4 : 5);
      const int LPR = 1 << lpr_log2, RPW = 32 >> lpr_log2;
      const int sub = lane >> lpr_log2, l = lane & (LPR - 1);
      const int stride = nw * RPW;
      int rho = warp * RPW + sub;
      int t = rho < r ? ptr[rho] : 0, te = rho < r ? ptr[rho + 1] : 0;
      int col[4]; double v[4];
#pragma unroll
      for (int u = 0; u < 4; u++) {
        const bool ok = t + u < te;
        v[u] = ok ? A.tt_val[t + u] : 0.0;
        col[u] = ok ? A.tt_col[t + u] : 0;
      }
      const int half = gw >> 1;
      double acc[4] = {0.0, 0.0, 0.0, 0.0};                      // vec: two double2 (chunks l, l + LPR); else 4 columns
      while (rho < r) {
        int nrho = rho, nt = t + 4, nte = te;
        if (nt >= te) { nrho = rho + stride; nt = nrho < r ? ptr[nrho] : 0; nte = nrho < r ? ptr[nrho + 1] : 0; }
        int ncol[4]; double nv[4];
#pragma unroll
        for (int u = 0; u < 4; u++) {
          const bool ok = nt + u < nte;
          nv[u] = ok ? A.tt_val[nt + u] : 0.0;
          ncol[u] = ok ? A.tt_col[nt + u] : 0;
        }
        if (vec) {
          double2 x[4][2];
#pragma unroll
          for (int u = 0; u < 4; u++) {
            const double2 *Dc = reinterpret_cast<const double2 *>(D + (long long)col[u] * n + c0);
            x[u][0] = l < half ? Dc[l] : make_double2(0.0, 0.0);
            x[u][1] = l + LPR < half ? Dc[l + LPR] : make_double2(0.0, 0.0);
          }
#pragma unroll
          for (int u = 0; u < 4; u++) {
            acc[0] += v[u] * x[u][0].x; acc[1] += v[u] * x[u][0].y;
            acc[2] += v[u] * x[u][1].x; acc[3] += v[u] * x[u][1].y;
          }
        } else {
          double x[4][4];
#pragma unroll
          for (int u = 0; u < 4; u++) {
            const double *Dc = D + (long long)col[u] * n + c0;
#pragma unroll
            for (int ch = 0; ch < 4; ch++) { const int c = l + LPR * ch; x[u][ch] = c < gw ? Dc[c] : 0.0; }
          }
#pragma unroll
          for (int u = 0; u < 4; u++)
#pragma unroll
            for (int ch = 0; ch < 4; ch++) acc[ch] += v[u] * x[u][ch];
        }
        if (nrho != rho) {
          if (vec) {
            double2 *dst = reinterpret_cast<double2 *>(Tt + (long long)rho * gwa);
            if (l < half) dst[l] = make_double2(acc[0], acc[1]);
            if (l + LPR < half) dst[l + LPR] = make_double2(acc[2], acc[3]);
          } else {
            double *dst = Tt + (long long)rho * gwa;
#pragma unroll
            for (int ch = 0; ch < 4; ch++) { const int c = l + LPR * ch; if (c < gw) dst[c] = acc[ch]; }
          }
#pragma unroll
          for (int ch = 0; ch < 4; ch++) acc[ch] = 0.0;
        }
        rho = nrho; t = nt; te = nte;
#pragma unroll
        for (int u = 0; u < 4; u++) { col[u] = ncol[u]; v[u] = nv[u]; }
      }
    }
    __syncthreads();
    if (P.mode != 0) {
      // ---------------- 2a. entry-wise evaluation on the strip's share of the needed set
      const int *pq = A.need_pq + PG.need_beg;
      const int g4 = tid & 3;
      const int e0 = A.tt_ptr[P.r0], e1 = A.tt_ptr[P.r0 + r];
      for (int u0 = 0; u0 < PG.need_cnt; u0 += STRIP_THREADS >> 2) {
        const int u = u0 + (tid >> 2);
        const bool live = u < PG.need_cnt;
        const int v = live ? pq[u] : 0, pp = v & 0xffff, qq = v >> 16;
        double acc = 0.0;
        if (P.mode == 1) {
          if (live) {
#pragma unroll 8
            for (int rho = g4; rho < r; rho += 4) acc += D[pp + (long long)R[rho] * n] * Tt[(qq - c0) + (long long)rho * gwa];
          }
        } else {
          if (live) {
#pragma unroll 8
            for (int t = e0 + g4; t < e1; t += 4)
              acc += A.tt_val[t] * (D[pp + (long long)A.tt_row[t] * n] * D[qq + (long long)A.tt_col[t] * n]);
          }
        }
        acc += __shfl_xor_sync(0xffffffffu, acc, 1);
        acc += __shfl_xor_sync(0xffffffffu, acc, 2);
        if (live && g4 == 0) Wg[(qq * (2 * n - qq + 1)) / 2 - qq + pp - Gp.base] = acc;
      }
    } else {
      // ---------------- 2b. W_strip = D(c0:n, R) T_strip on the strip's supertiles (rounds of 8 warps; the planner keeps
      // a strip at <= 8 supertiles whenever the entry cap allows it)
      const int nslab = (r + FKC - 1) / FKC;
      for (int it0 = Gp.item_beg; it0 < Gp.item_end; it0 += nw) {
        const bool have = it0 + warp < Gp.item_end;
        const int2 IJ = have ? A.items[it0 + warp] : make_int2(0, 0);
        const int rb = 32 * IJ.x, cb = 32 * IJ.y;
        const int nra = have ? min(4, (n - rb + 7) >> 3) : 0;
        const int ncb = have ? min(4, (n - cb + 7) >> 3) : 0;
        const bool diag = (IJ.x == IJ.y);
        const bool full = have && !diag && nra == 4 && ncb == 4;
        unsigned tmask = 0;
#pragma unroll
        for (int a = 0; a < 4; a++)
#pragma unroll
          for (int b = 0; b < 4; b++) if (a < nra && b < ncb && (!diag || a >= b)) tmask |= 1u << (a * 4 + b);
        double acc[4][4][2];
#pragma unroll
        for (int a = 0; a < 4; a++)
#pragma unroll
          for (int b = 0; b < 4; b++) { acc[a][b][0] = 0.0; acc[a][b][1] = 0.0; }
        // three-stage ring: slabs s+1 and s+2 are in flight while slab s feeds the tensor pipe
#pragma unroll
        for (int s = 0; s < STRIP_STAGES - 1; s++) {
          if (s < nslab) strip_stage(stA + s * FKC * A.ldA, stB + s * FKC * A.ldB, A.ldA, A.ldB, D, Tt, R, n, r, s * FKC, c0, gw, gwa, vec);
          cp_async_commit();
        }
        int buf = 0;
        for (int s = 0; s < nslab; s++) {
          cp_async_wait_group<STRIP_STAGES - 2>();
          __syncthreads();                                        // slab s visible; everyone is done with slab s-1
          {
            const int sn = s + STRIP_STAGES - 1;
            int bn = buf + STRIP_STAGES - 1; if (bn >= STRIP_STAGES) bn -= STRIP_STAGES;
            if (sn < nslab) strip_stage(stA + bn * FKC * A.ldA, stB + bn * FKC * A.ldB, A.ldA, A.ldB, D, Tt, R, n, r, sn * FKC, c0, gw, gwa, vec);
            cp_async_commit();
          }
          const double *As = stA + buf * FKC * A.ldA + (rb - c0) + qr, *Bs = stB + buf * FKC * A.ldB + (cb - c0) + qr;
          if (full) {
#pragma unroll
            for (int k4 = 0; k4 < FKC; k4 += 4) {
              double af[4], bf[4];
#pragma unroll
              for (int a = 0; a < 4; a++) af[a] = As[(k4 + qc) * A.ldA + 8 * a];
#pragma unroll
              for (int b = 0; b < 4; b++) bf[b] = Bs[(k4 + qc) * A.ldB + 8 * b];
#pragma unroll
              for (int a = 0; a < 4; a++)
#pragma unroll
                for (int b = 0; b < 4; b++) dmma_m8n8k4(acc[a][b][0], acc[a][b][1], af[a], bf[b]);
            }
          } else if (have) {
#pragma unroll
            for (int k4 = 0; k4 < FKC; k4 += 4) {
              double af[4], bf[4];
#pragma unroll
              for (int a = 0; a < 4; a++) af[a] = (a < nra) ? As[(k4 + qc) * A.ldA + 8 * a] : 0.0;
#pragma unroll
              for (int b = 0; b < 4; b++) bf[b] = (b < ncb) ? Bs[(k4 + qc) * A.ldB + 8 * b] : 0.0;
#pragma unroll
              for (int a = 0; a < 4; a++)
#pragma unroll
                for (int b = 0; b < 4; b++)
                  if (tmask & (1u << (a * 4 + b))) dmma_m8n8k4(acc[a][b][0], acc[a][b][1], af[a], bf[b]);
            }
          }
          if (++buf == STRIP_STAGES) buf = 0;
        }
        cp_async_wait_all();
#pragma unroll
        for (int a = 0; a < 4; a++)
#pragma unroll
          for (int b = 0; b < 4; b++)
#pragma unroll
            for (int e = 0; e < 2; e++) {
              const int p = rb + 8 * a + qr, q = cb + 8 * b + 2 * qc + e;
              if (a < nra && b < ncb && p < n && q < n && p >= q) Wg[(q * (2 * n - q + 1)) / 2 - q + p - Gp.base] = acc[a][b][e];
            }
        __syncthreads();
      }
    }
    __syncthreads();
    // ---------------- 3. partial inner products with the partners up to and including the pair's own constraint
    {
      double *part = A.ws + PG.part_off;
      switch (A.blk_lanes[P.k]) {
        case 4: strip_dots<4>(A, P, Wk.g, ng, Wg, part, warp, lane, nw); break;
        case 8: strip_dots<8>(A, P, Wk.g, ng, Wg, part, warp, lane, nw); break;
        case 16: strip_dots<16>(A, P, Wk.g, ng, Wg, part, warp, lane, nw); break;
        default: strip_dots<32>(A, P, Wk.g, ng, Wg, part, warp, lane, nw); break;
      }
    }
    if (tid == 0) s_w[turn ^ 1] = nxt;
    __syncthreads();                                            // Wg, sR / sPtr and the scratch slot are re-used
  }
}

// ADA(i, c) += sum over the pairs of c, over their strips (fixed order), of the partial inner products; absd likewise.
__global__ void __launch_bounds__(256)
ada3_strip_reduce_kernel(const long long *adajc, const int *adair, const int *invperm, int first, const int *cpair_beg,
                         const AdaPair *pairs, const int *blkp_beg, const BlkPartner *blkp, const int *blk_grp_beg,
                         const int *pair_pg, const StripPG *pg, const double *ws, double *ada, double *absd, int use_map, int m) {
  extern __shared__ int sred_slot[];
  const int c = blockIdx.x;
  const int pcb = cpair_beg[c], pce = cpair_beg[c + 1];
  if (pce == pcb) return;
  const int ipc = invperm[c];
  const long long colbeg = adajc[c];
  ColSlots cs{adair + colbeg, (int)(adajc[c + 1] - colbeg), nullptr};
  if (use_map) { build_slots(sred_slot, cs.rows, cs.collen, m); cs.slot = sred_slot; }
  if (threadIdx.x == 0) {
    const int sd = ipc >= first ? cs.find(c) : -1;
    absd[c] = sd >= 0 ? ada[colbeg + sd] : 0.0;
  }
  for (int pc = pcb; pc < pce; pc++) {
    __syncthreads();                               // two blocks can feed the same entry: keep them in order
    const AdaPair P = pairs[pc];
    const int ng = blk_grp_beg[P.k + 1] - blk_grp_beg[P.k];
    const StripPG *G = pg + pair_pg[pc];
    const int tb = blkp_beg[P.k];
    for (int t = threadIdx.x; t <= P.rank; t += blockDim.x) {
      const int i = blkp[tb + t].j;
      const int sl = cs.find(i);
      if (sl < 0) continue;
      double s = 0.0;
      for (int g = 0; g < ng; g++) if (G[g].part_off >= 0) s += ws[G[g].part_off + t];
      ada[colbeg + sl] += s;
      if (t == P.rank && ipc >= first) {
        double a = 0.0;
        for (int g = 0; g < ng; g++) if (G[g].part_off >= 0) a += ws[G[g].part_off + P.rank + 1];
        absd[c] += a;
      }
    }
  }
}

__global__ void gather_val_kernel(long long n, const int *src, const double *Atpr, double *val) {
  for (long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x; t < n; t += (long long)gridDim.x * blockDim.x) val[t] = Atpr[src[t]];
}

}  // namespace sb
