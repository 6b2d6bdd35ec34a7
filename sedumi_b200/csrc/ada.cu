// ada.cu -- assembly of the Schur complement ADA' = A D(d^2) A' (getada1 / getada2 / getada3).
//
// Reference semantics:
//   getada1.c:89-152   LP + Lorentz-det part: ada(i,j) = sum_r a_ri dsqr_r a_rj over rows < start of
//                      PSD, dsqr = [d.l; -d.det; det_k on the norm-bound rows of cone k]; written only
//                      where invperm[i] <= invperm[j] ("upper triangle in perm order"), zero elsewhere,
//                      and only for columns that have LP/Lorentz nonzeros
//   getada2.c:74-118   ada += DAt.q' * DAt.q on the entries that are upper in Aord.qperm order
//   getada3.c:253-361  PSD part: ada(i,j) += <A_i, D A_j D> on entries upper in Aord.sperm order,
//                      absd(j) = ada_in(j,j) + sum |a_j .* vec(D A_j D)| (0 for the leading constraints
//                      of sperm that have no PSD nonzeros, :282-284), then ADA := ADA+ADA'-diag (:151-180)
//
// GPU design for the PSD part.  The reference walks constraints in a greedy order and evaluates
// vec(D A_j D) only on an incrementally growing pattern with BLAS-1 dots (spscale.c:249-305).  That
// is a scalar algorithm.  Here each (constraint j, PSD block k) pair with nonzeros becomes one dense
// product   W_jk = D_k * sym(A_jk) * D_k = D_k(:,R) * [sym(A_jk)(R,:) D_k]   (R = nonzero rows of
// sym(A_jk)), run as a batched DMMA tile GEMM over ALL pairs of a batch in one launch (gemm.cuh),
// followed by one warp per ADA entry that dots the sparse A_ik against W_jk over the blocks i and j
// share.  One writer per entry: deterministic, no atomics.  absd and the symmetrisation ride along.
#include <algorithm>
#include <map>
#include "gemm.cuh"
#include <chrono>
#include "sb_internal.h"

namespace sb {

struct AdaPair {      // one (constraint, PSD block) with nonzeros
  int j, k;           // constraint, block
  int e0, e1;         // entries [e0,e1) in ent_*
  int r0, r;          // rows R: Rlist[r0 .. r0+r)
  long long tt_off;   // offset of Tt (n x r) in the batch workspace
  long long w_off;    // offset of W in the batch workspace: n x n (dense mode) or |U_k| values (sparse mode)
  int sparse;         // 1: W is only evaluated on U_k, the union pattern of block k
  int rank;           // position of this pair in its block's partner list (sparsest constraint first)
  long long part_off; // constraints with several blocks: offset of this pair's partial sums (npartners(k)+1)
  long long fpart_off; // the same in the compact workspace of the fused path (no T / W there)
  // fused path: how W_jk is evaluated.  A pair only needs W on the union of the patterns of the partners that precede
  // it in its block's list (the observation behind the reference's incremental `dz`, getada3.c:305-326): when that
  // set is small, W is evaluated entry by entry there (mode 1: through T, mode 2: directly from the few entries of
  // A_jk) instead of as a dense DMMA product (mode 0).
  int mode, need_cnt;
  long long need_off;
  long long slot_off;  // fused path: position in column j of ADA of every partner up to this pair's rank (or -1), looked up at plan time
};

// --------------------------------------------------------------------- sparse A'WA on a pattern
// One CTA per ADA column c; one warp per stored entry (i,c).  B is CSC with per-column row ranges
// [lo[col], hi[col]).  out = (accumulate ? in : 0) + sum_r B(r,i) w(r) B(r,c)  where pred holds;
// elsewhere out = accumulate ? in : 0.  Columns with an empty range are skipped when skip_empty.
__global__ void __launch_bounds__(256)
ata_pattern_kernel(int m, const long long *adajc, const int *adair, const long long *lo, const long long *hi,
                   const int *Bir, const double *Bpr, const double *w, const int *invperm,
                   const double *in, double *out, int accumulate, int skip_empty) {
  const int c = blockIdx.x;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = blockDim.x >> 5;
  const long long clo = lo[c], chi = hi[c];
  const int ipc = invperm[c];
  const bool empty_c = skip_empty && (clo >= chi);
  if (empty_c) {                                     // nothing to add in this column: a coalesced copy / clear
    for (long long inz = adajc[c] + threadIdx.x; inz < adajc[c + 1]; inz += blockDim.x) out[inz] = accumulate ? in[inz] : 0.0;
    return;
  }
  for (long long inz = adajc[c] + warp; inz < adajc[c + 1]; inz += nw) {
    const int i = adair[inz];
    double base = accumulate ? in[inz] : 0.0;
    if (empty_c || invperm[i] > ipc) { if (lane == 0) out[inz] = base; continue; }
    long long alo = lo[i], ahi = hi[i], blo = clo, bhi = chi;
    if (ahi - alo > bhi - blo) { long long t = alo; alo = blo; blo = t; t = ahi; ahi = bhi; bhi = t; }
    double acc = 0.0;
    for (long long p = alo + lane; p < ahi; p += 32) {
      int r = Bir[p];
      long long l = blo, h = bhi;
      while (l < h) { long long mid = (l + h) >> 1; if (Bir[mid] < r) l = mid + 1; else h = mid; }
      if (l < bhi && Bir[l] == r) acc += Bpr[p] * (w ? w[r] : 1.0) * Bpr[l];
    }
    for (int o = 16; o > 0; o >>= 1) acc += __shfl_down_sync(0xffffffffu, acc, o);
    if (lane == 0) out[inz] = base + acc;
  }
}

// dsqr = [d.l ; -d.det ; det_k repeated over the norm-bound rows of Lorentz cone k]   (getada1.c:110-119)
__global__ void dsqr_kernel(int lpN, int nq, const long long *qstart, const double *dl, const double *ddet, double *dsqr) {
  // qstart[k], k=0..nq: 0-based first norm-bound row of cone k (qstart[0] = lpN + nq)
  long long tot = nq ? qstart[nq] : lpN;
  for (long long r = blockIdx.x * (long long)blockDim.x + threadIdx.x; r < tot; r += (long long)gridDim.x * blockDim.x) {
    double v;
    if (r < lpN) v = dl[r];
    else if (r < lpN + nq) v = -ddet[r - lpN];
    else {
      int l = 0, h = nq;                          // last k with qstart[k] <= r
      while (h - l > 1) { int mid = (l + h) >> 1; if (qstart[mid] <= r) l = mid; else h = mid; }
      v = ddet[l];
    }
    dsqr[r] = v;
  }
}

// ---- dense route for B'WB when B is (nearly) full (nb.mat: 66 % of At is nonzero; getada.m itself switches
// to full storage above 20 %, getada.m:27-34): Bd(i, r) = B(r0 + r, i) as an m x R matrix, the product
// in K-chunks on the DMMA engine, and a gather onto the ADA pattern that adds the chunks in order.
__global__ void dense_from_csc_kernel(int m, const long long *lo, const long long *hi, const int *Bir, const double *Bpr,
                                      long long r0, long long R, double *Bd) {
  const int c = blockIdx.x;
  for (long long p = lo[c] + threadIdx.x; p < hi[c]; p += blockDim.x) {
    const long long r = Bir[p] - r0;
    if (r >= 0 && r < R) Bd[c + r * m] = Bpr[p];
  }
}
__global__ void scale_cols_kernel(long long tot, int m, const double *w, const double *Bd, double *Bw) {
  for (long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x; idx < tot; idx += (long long)gridDim.x * blockDim.x)
    Bw[idx] = Bd[idx] * w[idx / m];
}
__global__ void __launch_bounds__(256)
gather_dense_kernel(int m, const long long *adajc, const int *adair, const int *invperm, const double *Cp, int nchunk,
                    const double *in, double *out, int accumulate) {
  const int c = blockIdx.x;
  const int ipc = invperm[c];
  for (long long inz = adajc[c] + threadIdx.x; inz < adajc[c + 1]; inz += blockDim.x) {
    const int i = adair[inz];
    double v = accumulate ? in[inz] : 0.0;
    if (invperm[i] <= ipc) {
      double acc = 0.0;
      for (int p = 0; p < nchunk; p++) acc += Cp[(long long)p * m * m + i + (long long)c * m];
      v += acc;
    }
    out[inz] = v;
  }
}

// udsqr as it arrives ([vec Re D; vec Im D] for Hermitian blocks) -> the embedded blocks [[Re,-Im],[Im,Re]]
__global__ void ada_embed_d_kernel(const int *nraw, const int *cplx, const long long *rawoff, const long long *emboff,
                                   const double *raw, double *emb) {
  const int k = blockIdx.y, n = nraw[k], c = cplx[k], ne = c ? 2 * n : n;
  const double *re = raw + rawoff[k], *im = re + (long long)n * n;
  double *E = emb + emboff[k];
  const long long tot = (long long)n * n;
  for (long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x; idx < tot; idx += (long long)gridDim.x * blockDim.x) {
    const int p = (int)(idx % n), q = (int)(idx / n);
    const double zr = re[idx];
    E[p + (long long)q * ne] = zr;
    if (c) {
      const double zi = im[idx];
      E[(p + n) + (long long)(q + n) * ne] = zr;
      E[(p + n) + (long long)q * ne] = zi;
      E[p + (long long)(q + n) * ne] = -zi;
    }
  }
}

// getDAtm.m:40-43:  DAt.q(k,j) = d.q1(k) * A(trace row of cone k, j) + sum_{i in norm rows of cone k} d.q2(i) * A(i,j).
// The pattern (one entry per (column, Lorentz cone touched)) is compiled into the plan; WIDE = one warp
// per entry (long cones), otherwise one thread per entry.
template <bool WIDE>
__global__ void datq_kernel(long long nent, const int *cone, const int *tsrc, const long long *lo, const long long *hi,
                            const int *Air, const double *Atpr, const double *q1, const double *q2, long long q2row0, double *out) {
  const long long gid = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  const long long e = WIDE ? (gid >> 5) : gid;
  if (e >= nent) return;
  const int lane = threadIdx.x & 31;
  double acc = 0.0;
  if (WIDE) {
    for (long long p = lo[e] + lane; p < hi[e]; p += 32) acc += q2[Air[p] - q2row0] * Atpr[p];
    for (int o = 16; o > 0; o >>= 1) acc += __shfl_down_sync(0xffffffffu, acc, o);
    if (lane != 0) return;
  } else {
    for (long long p = lo[e]; p < hi[e]; p++) acc += q2[Air[p] - q2row0] * Atpr[p];
  }
  const int t = tsrc[e];
  out[e] = (t >= 0 ? q1[cone[e]] * Atpr[t] : 0.0) + acc;
}

// --------------------------------------------------------------------- getada3 kernels
// Tt_p(c, rho) = (D_k * sym(A_jk))(c, R[rho]) = sum over the entries of column R[rho] of sym(A_jk).
// One CTA per pair, one thread per element (c, rho); the per-column entry lists (D column, weight,
// source of the value in At.pr) are compiled into the plan, so there is no read-modify-write.
__global__ void __launch_bounds__(256)
build_tt_kernel(const AdaPair *pairs, int p0, const int *blk_n, const long long *blk_off,
                const int *tt_ptr, const int *tt_col, const int *tt_src, const double *tt_w,
                const double *Atpr, const double *udsqr, double *ws) {
  const AdaPair P = pairs[p0 + blockIdx.x];
  const int n = blk_n[P.k];
  const double *D = udsqr + blk_off[P.k];
  double *Tt = ws + P.tt_off;
  const int *ptr = tt_ptr + P.r0;                  // P.r + 1 entries are readable: ptr[rho] .. ptr[rho+1]
  for (int idx = threadIdx.x; idx < n * P.r; idx += blockDim.x) {
    const int c = idx % n, rho = idx / n;
    double acc = 0.0;
    for (int t = ptr[rho]; t < ptr[rho + 1]; t++)
      acc += (tt_w[t] * Atpr[tt_src[t]]) * D[c + (long long)tt_col[t] * n];
    Tt[idx] = acc;
  }
}

// Sparse mode (blocks whose constraints touch only a small part of the n x n block, e.g. MaxCut where
// A_j = e_j e_j'): W_j is needed only on U_k = union of the patterns of all A_ik -- the same observation
// the reference exploits with its incremental `dz` pattern (getada3.c:305-326).  One thread per (pair, u):
//   W_j(p_u,q_u) = sum_rho D(p_u, R[rho]) * Tt(q_u, rho)
__global__ void __launch_bounds__(256)
sparse_w_kernel(const AdaPair *pairs, int p0, int npairs, const int *blk_n, const long long *blk_off, const int *ublk_off,
                const int *u_p, const int *u_q, const int *Rlist, const double *udsqr, double *ws) {
  for (int pi = blockIdx.y; pi < npairs; pi += gridDim.y) {
    const AdaPair P = pairs[p0 + pi];
    if (!P.sparse) continue;
    const int n = blk_n[P.k];
    const int u0 = ublk_off[P.k], nu = ublk_off[P.k + 1] - u0;
    const double *D = udsqr + blk_off[P.k];
    const double *Tt = ws + P.tt_off;
    double *W = ws + P.w_off;
    const int *R = Rlist + P.r0;
    for (int u = blockIdx.x * blockDim.x + threadIdx.x; u < nu; u += gridDim.x * blockDim.x) {
      const int pp = u_p[u0 + u], qq = u_q[u0 + u];
      double acc = 0.0;
      for (int rho = 0; rho < P.r; rho++) acc += D[pp + (long long)R[rho] * n] * Tt[qq + (long long)rho * n];
      W[u] = acc;
    }
  }
}

// <A_ik, W_ck> for every stored ADA entry.  One CTA per (constraint c, PSD block k) pair: W_ck is staged
// in shared memory (packed lower triangle, or its values on U_k in sparse mode; read in place when it
// does not fit) and every constraint i of block k with invperm(i) <= invperm(c) takes its inner
// product from there, a group of G lanes per partner.  Constraints that live in ONE block write
// ADA(i,c) directly (nobody else touches column c); constraints spanning several blocks write
// per-pair partial sums that ada3_reduce_kernel adds in block order -- deterministic, no atomics.
// (Replaces the reference's per-entry accumulation, getada3.c:198-268.)
struct BlkPartner { int j, e0, e1, src0; };          // src0 = ent_src[e0]: first At.pr index of the pair

struct ColSlots {        // row -> position inside one ADA column: shared-memory map, or binary search
  const int *rows; int collen; const int *slot;
  __device__ int find(int i) const {
    if (slot) return slot[i];
    int l = 0, h = collen;
    while (l < h) { int mid = (l + h) >> 1; if (rows[mid] < i) l = mid + 1; else h = mid; }
    return (l < collen && rows[l] == i) ? l : -1;
  }
};

__device__ __forceinline__ void build_slots(int *slot, const int *rows, int collen, int m) {
  for (int t = threadIdx.x; t < m; t += blockDim.x) slot[t] = -1;
  __syncthreads();
  for (int t = threadIdx.x; t < collen; t += blockDim.x) slot[rows[t]] = t;
  __syncthreads();
}

struct DotsCtx {
  AdaPair P; int c, ipc, first, multi, warp, lane, nw;
  int rank_limit;     // >= 0: the partners are the first rank_limit+1 entries of the block's list; < 0: filter by invperm
  long long colbeg;
  ColSlots cs;
  const int *eidx; const double *Wp;
  const int *blkp_beg; const BlkPartner *blkp; const int *invperm;
  const double *Atpr; const int *ent_src; const double *ent_scale;
  double *ws, *ada, *absd;
  const int *slot_tab;   // by_rank: slot_tab[t - tb] = position of partner t's row in ADA column c (else nullptr: search)
};
// The partner loop with G lanes per partner; G is chosen PER BLOCK from the average number of entries of its pairs
// (control07: 161 entries per pair in the 70x70 block, exactly 1 in the 35x35 block).
template <int G>
__device__ __forceinline__ void dots_partners(const DotsCtx &X) {
  const AdaPair &P = X.P;
  const int c = X.c, ipc = X.ipc, first = X.first, warp = X.warp, lane = X.lane, nw = X.nw;
  const bool multi = X.multi;
  const long long colbeg = X.colbeg;
  const ColSlots &cs = X.cs;
  const int *eidx = X.eidx; const double *Wp = X.Wp;
  const int *blkp_beg = X.blkp_beg; const BlkPartner *blkp = X.blkp; const int *invperm = X.invperm;
  const double *Atpr = X.Atpr; const int *ent_src = X.ent_src; const double *ent_scale = X.ent_scale;
  double *ws = X.ws, *ada = X.ada, *absd = X.absd;
  constexpr int GPW = 32 / G;                      // partner groups per warp
  const int grp = lane / G, gl = lane % G;
  const unsigned gmask = G == 32 ? 0xffffffffu : (((1u << G) - 1u) << (grp * G));   // groups diverge: sync only the group
  const int tb = blkp_beg[P.k], te = blkp_beg[P.k + 1];
  const bool by_rank = X.rank_limit >= 0;
  const int tl = by_rank ? tb + X.rank_limit + 1 : te;      // end of the partner loop
  double *part = ws + P.part_off;                 // multi: one partial per partner, then the |.| sum of the diagonal
  // the descriptor and the order of the NEXT partner are fetched while the current one is worked on: the chain
  // descriptor -> invperm -> entries -> W is four dependent loads, which bounded this loop
  int t = tb + warp * GPW + grp;
  BlkPartner Qn = t < tl ? blkp[t] : BlkPartner{0, 0, 0, 0};
  int ipn = (t < tl && !by_rank) ? invperm[Qn.j] : 0;
  for (; t < tl; t += nw * GPW) {
    const BlkPartner Q = Qn;
    const int ipi = ipn;
    {
      const int tn = t + nw * GPW;
      if (tn < tl) { Qn = blkp[tn]; ipn = by_rank ? 0 : invperm[Qn.j]; }
    }
    if (!by_rank && ipi > ipc) continue;
    // the partner's position in ADA column c: a table built with the plan (a binary search over a 5000-row column is
    // 12 dependent L2 round trips on the lane that writes the result: 11 % of the fused kernel's stall samples)
    const int sl_tab = X.slot_tab ? X.slot_tab[t - tb] : -2;
    const double *av = Atpr + Q.src0 - Q.e0;            // the entries of one pair are consecutive in At.pr ...
    double acc = 0.0, aabs = 0.0;
    int e = Q.e0 + gl;
    if (ent_scale) {                                    // ... except with Hermitian blocks (embedded entries, signs)
      for (; e < Q.e1; e += G) {
        const double term = (Atpr[ent_src[e]] * ent_scale[e]) * Wp[eidx[e]];
        acc += term;
        aabs += fabs(term);
      }
    }
    // trips of 8 entries per lane, all 16 loads of a trip issued before the first product (a partner with up to 8 G
    // entries costs one L2 round trip); lanes beyond the end contribute an explicit zero -- W may hold entries that were
    // never written (entry-wise pairs), so 0 * W is not safe
    for (; e < Q.e1; e += 8 * G) {
      double a[8]; int ix[8];
#pragma unroll
      for (int u = 0; u < 8; u++) {
        const bool ok = e + u * G < Q.e1;
        a[u] = ok ? av[e + u * G] : 0.0;
        ix[u] = ok ? eidx[e + u * G] : -1;
      }
#pragma unroll
      for (int u = 0; u < 8; u++) {
        const double term = ix[u] >= 0 ? a[u] * Wp[ix[u]] : 0.0;
        acc += term; aabs += fabs(term);
      }
    }
#pragma unroll
    for (int o = G / 2; o > 0; o >>= 1) {
      acc += __shfl_down_sync(gmask, acc, o, G);
      aabs += __shfl_down_sync(gmask, aabs, o, G);
    }
    if (gl == 0) {
      if (multi) {
        part[t - tb] = acc;
        if (Q.j == c) part[te - tb] = aabs;
      } else {
        const int sl = sl_tab != -2 ? sl_tab : cs.find(Q.j);
        if (sl >= 0) {
          ada[colbeg + sl] += acc;
          if (Q.j == c && ipc >= first) absd[c] += aabs;
        }
      }
    }
  }
}

__global__ void __launch_bounds__(256)
ada3_dots_kernel(int p0, const long long *adajc, const int *adair, const int *invperm, int first,
                 const int *cpair_beg, const AdaPair *pairs, const int *blk_n, const int *ublk_off,
                 const int *blkp_beg, const BlkPartner *blkp,
                 const int *ent_lin, const int *ent_pk, const int *ent_src, const double *Atpr, const double *ent_scale,
                 double *ws, double *ada, double *absd, int wcap, int use_map, int m, const int *blk_group) {
  extern __shared__ double dots_sm[];
  double *Wsm = dots_sm;
  int *slot = (int *)(dots_sm + wcap);
  const AdaPair P = pairs[p0 + blockIdx.x];
  const int c = P.j;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, nw = blockDim.x >> 5;
  const bool multi = cpair_beg[c + 1] - cpair_beg[c] > 1;
  const int ipc = invperm[c];
  const long long colbeg = adajc[c];
  ColSlots cs{adair + colbeg, (int)(adajc[c + 1] - colbeg), nullptr};
  if (!multi) {
    if (use_map) { build_slots(slot, cs.rows, cs.collen, m); cs.slot = slot; }
    if (tid == 0) {
      const int sd = ipc >= first ? cs.find(c) : -1;
      absd[c] = sd >= 0 ? ada[colbeg + sd] : 0.0;
    }
  }
  const int n = blk_n[P.k];
  const double *Wg = ws + P.w_off;
  const int wsize = P.sparse ? (ublk_off[P.k + 1] - ublk_off[P.k]) : n * (n + 1) / 2;
  const bool stage = wsize <= wcap;
  if (stage) {
    if (P.sparse) for (int t = tid; t < wsize; t += blockDim.x) Wsm[t] = Wg[t];
    else
      for (int q = warp; q < n; q += nw) {
        const double *src = Wg + (long long)q * n;
        double *dst = Wsm + ((long long)q * (2 * n - q + 1)) / 2 - q;       // packed column q, indexed by row p >= q
        for (int pp = q + lane; pp < n; pp += 32) dst[pp] = src[pp];
      }
  }
  __syncthreads();
  const int *eidx = stage ? ent_pk : ent_lin;
  const double *Wp = stage ? Wsm : Wg;
  DotsCtx X;
  X.P = P; X.c = c; X.ipc = ipc; X.first = first; X.multi = multi ? 1 : 0; X.warp = warp; X.lane = lane; X.nw = nw;
  X.rank_limit = -1; X.slot_tab = nullptr;
  X.colbeg = colbeg; X.cs = cs; X.eidx = eidx; X.Wp = Wp; X.blkp_beg = blkp_beg; X.blkp = blkp; X.invperm = invperm;
  X.Atpr = Atpr; X.ent_src = ent_src; X.ent_scale = ent_scale; X.ws = ws; X.ada = ada; X.absd = absd;
  switch (blk_group[P.k]) {
    case 4: dots_partners<4>(X); break;
    case 8: dots_partners<8>(X); break;
    case 16: dots_partners<16>(X); break;
    default: dots_partners<32>(X); break;
  }
}

// Constraints spanning several PSD blocks: add the per-pair partial sums into column c, block by block.
__global__ void __launch_bounds__(256)
ada3_reduce_kernel(int c0, const long long *adajc, const int *adair, const int *invperm, int first,
                   const int *cpair_beg, const AdaPair *pairs, const int *blkp_beg, const BlkPartner *blkp,
                   const double *ws, double *ada, double *absd, int use_map, int m, int fused) {
  extern __shared__ int red_slot[];
  const int c = c0 + blockIdx.x;
  const int pcb = cpair_beg[c], pce = cpair_beg[c + 1];
  if (pce - pcb <= 1) return;
  const int ipc = invperm[c];
  const long long colbeg = adajc[c];
  ColSlots cs{adair + colbeg, (int)(adajc[c + 1] - colbeg), nullptr};
  if (use_map) { build_slots(red_slot, cs.rows, cs.collen, m); cs.slot = red_slot; }
  if (threadIdx.x == 0) {
    const int sd = ipc >= first ? cs.find(c) : -1;
    absd[c] = sd >= 0 ? ada[colbeg + sd] : 0.0;
  }
  for (int pc = pcb; pc < pce; pc++) {
    __syncthreads();                               // two blocks can feed the same entry: keep them in order
    const int k = pairs[pc].k;
    const double *part = ws + (fused ? pairs[pc].fpart_off : pairs[pc].part_off);
    const int tb = blkp_beg[k], te = blkp_beg[k + 1];
    const int tl = fused ? tb + pairs[pc].rank + 1 : te;     // fused path: the partners are a prefix of the block's list
    for (int t = tb + threadIdx.x; t < tl; t += blockDim.x) {
      const int i = blkp[t].j;
      if (!fused && invperm[i] > ipc) continue;
      const int sl = cs.find(i);
      if (sl < 0) continue;
      ada[colbeg + sl] += part[t - tb];
      if (i == c && ipc >= first) absd[c] += part[te - tb];
    }
  }
}

// absd for constraints without any pair (no kernel column above touches them): diag or 0.
__global__ void absd_nopsd_kernel(int m, const long long *adajc, const int *adair, const int *invperm, int first,
                                  const int *cpair_beg, const double *ada, double *absd, int all_diag) {
  int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= m) return;
  if (!all_diag && cpair_beg[c] < cpair_beg[c + 1]) return;      // handled by ada3_dots_kernel
  double v = 0.0;
  if (all_diag || invperm[c] >= first) {
    long long l = adajc[c], h = adajc[c + 1];
    while (l < h) { long long mid = (l + h) >> 1; if (adair[mid] < c) l = mid + 1; else h = mid; }
    if (l < adajc[c + 1] && adair[l] == c) v = ada[l];
  }
  absd[c] = v;
}

// X := X + X' - diag(X) on a full symmetric pattern (spmakesym, getada3.c:151-180).
__global__ void makesym_kernel(int m, const long long *jc, const int *ir, double *x) {
  const int c = blockIdx.x;
  for (long long inz = jc[c] + threadIdx.x; inz < jc[c + 1]; inz += blockDim.x) {
    const int i = ir[inz];
    if (i <= c) continue;                            // the strictly-lower entry owns the pair
    long long l = jc[i], h = jc[i + 1];
    while (l < h) { long long mid = (l + h) >> 1; if (ir[mid] < c) l = mid + 1; else h = mid; }
    if (l < jc[i + 1] && ir[l] == c) { double s = x[inz] + x[l]; x[inz] = s; x[l] = s; }
  }
}

// tt_val[t] = weight * value of the At entry it comes from (refreshed whenever the values of At change)
__global__ void tt_val_kernel(long long n, const double *tt_w, const int *tt_src, const double *Atpr, double *tt_val) {
  for (long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x; t < n; t += (long long)gridDim.x * blockDim.x)
    tt_val[t] = tt_w[t] * Atpr[tt_src[t]];
}

}  // namespace sb

#include "ada_fused.cuh"
#include "ada_strip.cuh"

using namespace sb;

struct sb200_ada_plan {
  int m = 0;
  long long N = 0, nnzA = 0, nnzADA = 0;
  int lpN = 0, nq = 0, nblk = 0;
  long long lq_rows = 0;          // rows before the PSD part covered by dsqr
  std::vector<int> blk_n, blk_nraw, blk_cplx; std::vector<long long> blk_off, blk_start, blk_rawoff;
  bool herm = false; long long lenud_emb = 0, lenud_raw = 0;
  DevBuf<double> d_De, d_ent_scale;
  DevBuf<int> d_blk_nraw, d_blk_cplx; DevBuf<long long> d_blk_rawoff;
  std::vector<AdaPair> pairs;
  std::vector<int> cpair_beg;
  struct Batch { int p0, p1, c0, c1; long long ws; int tile0, ntiles; int nsparse; int nmulti; };
  std::vector<Batch> batches;
  long long ws_max = 0;
  Hash128 key, val_hash;
  int pins = 0;                   // device-resident owners (sb200_ada_plan_retain); pinned plans are never evicted
  uint64_t cache_stamp = 0;
  bool have_vals = false;
  // device
  DevBuf<long long> d_Ajc, d_Ajc1, d_Ajcend, d_adajc, d_qstart, d_blk_off;
  DevBuf<int> d_Air, d_adair, d_blk_n, d_cpair_beg, d_ent_lin, d_ent_src, d_Rlist, d_tt_ptr, d_tt_col, d_tt_src, d_tt_row;
  DevBuf<double> d_tt_w;
  DevBuf<int> d_ublk_off, d_u_p, d_u_q, d_blkp_beg, d_ent_pk;
  DevBuf<BlkPartner> d_blkp;
  int wcap = 0, use_map = 0, dots_group = 32;
  DevBuf<int> d_blk_group;
  size_t dots_smem = 0;
  std::vector<int> blk_sparse;
  int max_nu = 0;
  DevBuf<AdaPair> d_pairs;
  // dense route (B'WB with nearly full B)
  struct DenseSet { long long R = 0; int nchunk = 0, ntiles = 0; DevBuf<GemmDesc> descs; DevBuf<GemmTile> tiles; };
  std::map<long long, DenseSet *> dense_sets;
  DevBuf<double> d_Bd_lq, d_Bd, d_Bw, d_Cp;
  long long cap_Bd = 0, cap_Cp = 0;
  bool lq_dense = false, lq_dense_valid = false;
  // DAt.q (nq x m CSC, pattern fixed by At): getDAtm on the device
  long long dq_nnz = 0; bool dq_wide = false;
  DevBuf<long long> d_dq_jc, d_dq_lo, d_dq_hi;
  DevBuf<int> d_dq_ir, d_dq_tsrc;
  DevBuf<double> d_dq_pr;
  DevBuf<GemmDesc> d_descs;
  DevBuf<GemmTile> d_tiles;
  DevBuf<double> d_Atpr, d_dsqr, d_ws;
  DevBuf<int> d_invperm, d_ident;
  // fused path (ada_fused.cuh): every block in dense mode and of order <= FUSED_MAX_N, no Hermitian block
  bool fused_ok = false, tt_val_valid = false;
  int fused_threads = 0, fused_grid = 0, fused_wcap = 0, fused_ldmax = 0, fused_small = 0;
  size_t fused_smem = 0;
  long long fused_scratch_stride = 0, fws = 0, n_tt = 0;
  int any_multi = 0;
  DevBuf<double> d_tt_val, d_fscratch, d_fws;
  DevBuf<int> d_fcounter, d_fitem_beg, d_fneed, d_forder, d_fslot;
  // row-wise (CSR) view of the pattern of At for products At*p without atomics (pcg.cu)
  DevBuf<long long> d_rowptr; DevBuf<int> d_rowcol, d_rowsrc;
  std::vector<long long> h_Ajc; std::vector<int> h_Air;
  bool csr_built = false;
  DevBuf<int2> d_fitems;
  long long fused_ndense = 0;
  DevBuf<unsigned long long> d_fprof; bool fprof_on = false;
  // strip path (ada_strip.cuh): blocks too large for two resident CTAs of the fused kernel
  bool strip_ok = false;
  int strip_grid = 0, strip_ldA = 0, strip_ldB = 0, strip_nwork = 0;
  size_t strip_smem = 0;
  long long strip_scratch_stride = 0, strip_nent = 0;
  DevBuf<StripGroup> d_sgroups; DevBuf<StripPG> d_spg; DevBuf<StripWork> d_swork;
  DevBuf<int> d_sblk_grp_beg, d_spair_pg, d_sblk_feoff, d_sfe_ptr, d_sfe_src, d_sneed, d_sblk_lanes;
  DevBuf<int2> d_sitems;
  DevBuf<unsigned short> d_sfe_pk;
  DevBuf<double> d_sfe_val, d_sscratch, d_sws;
};

static std::map<Hash128, sb200_ada_plan *> g_ada_plans;
static uint64_t g_ada_clock = 0;

static int ada_build(sb200_ada_plan *pl, sb_idx N, sb_idx m, const sb_idx *Ajc, const sb_idx *Air, const sb_idx *Ajc1,
                     sb_idx lpN, sb_idx nq, const sb_idx *qstart, sb_idx nblk, sb_idx nreal, const sb_idx *blkstart, const sb_idx *blkn,
                     const sb_idx *adajc, const sb_idx *adair) {
  pl->m = (int)m; pl->N = N; pl->nnzA = Ajc[m]; pl->nnzADA = adajc[m];
  pl->h_Ajc.assign(Ajc, Ajc + m + 1);
  pl->lpN = (int)lpN; pl->nq = (int)nq; pl->nblk = (int)nblk;
  SB_CHECK(pl->nnzA < 2147483647LL, "At has too many nonzeros for 32-bit entry indices");
  // Hermitian blocks (k >= nreal) are handled through the real embedding E(Z) = [[Re Z, -Im Z],[Im Z, Re Z]] of
  // order 2n: blk_n / blk_off describe the EMBEDDED blocks, blk_nraw / blk_rawoff the layout of udsqr as it arrives.
  long long off = 0, rawoff = 0;
  pl->herm = nreal < nblk;
  for (sb_idx k = 0; k < nblk; k++) {
    const int cplx = k >= nreal;
    const long long ne = cplx ? 2 * blkn[k] : blkn[k];
    SB_CHECK(ne < 46340, "PSD block order %lld out of range", (long long)blkn[k]);
    pl->blk_n.push_back((int)ne); pl->blk_off.push_back(off); pl->blk_start.push_back(blkstart[k]);
    pl->blk_nraw.push_back((int)blkn[k]); pl->blk_cplx.push_back(cplx); pl->blk_rawoff.push_back(rawoff);
    off += ne * ne; rawoff += (cplx ? 2 : 1) * blkn[k] * blkn[k];
  }
  pl->lenud_emb = off; pl->lenud_raw = rawoff;
  const long long psd0 = nblk ? blkstart[0] : N;
  pl->lq_rows = nq ? qstart[nq] : lpN;
  // ---- pairs
  std::vector<int> ent_p, ent_q, ent_lin, ent_src, Rlist, tt_ptr, tt_col, tt_row, tt_src;
  std::vector<double> ent_sgn;
  std::vector<double> tt_w;
  std::vector<std::vector<std::pair<int, std::pair<int, double>>>> percol;
  pl->cpair_beg.assign(m + 1, 0);
  std::vector<int> tmpR;
  for (sb_idx j = 0; j < m; j++) {
    pl->cpair_beg[j] = (int)pl->pairs.size();
    sb_idx inz = nblk ? Ajc1[j] : Ajc[j + 1];       // no PSD cone: nothing beyond the LP/Lorentz part matters
    SB_CHECK(Ajc1[j] >= Ajc[j] && Ajc1[j] <= Ajc[j + 1] && inz >= Ajc[j] && inz <= Ajc[j + 1], "getada3: Ajc1(%lld) outside its column", (long long)j);
    while (inz < Ajc[j + 1]) {
      sb_idx row = Air[inz];
      SB_CHECK(row >= psd0 && row < N, "getada3: row %lld of At is not in the PSD part", (long long)row);
      int k = (int)(std::upper_bound(pl->blk_start.begin(), pl->blk_start.end(), (long long)row) - pl->blk_start.begin()) - 1;
      const long long bs = pl->blk_start[k]; const int n = pl->blk_n[k];     // n: embedded order
      const int nr = pl->blk_nraw[k], cplx = pl->blk_cplx[k];
      const long long span = (long long)(cplx ? 2 : 1) * nr * nr;
      SB_CHECK(row < bs + span, "getada3: row %lld beyond PSD block %d", (long long)row, k);
      AdaPair P{}; P.j = (int)j; P.k = k; P.e0 = (int)ent_p.size();
      tmpR.clear();
      auto add_entry = [&](int p, int q, double sg) {
        ent_p.push_back(p); ent_q.push_back(q); ent_src.push_back((int)inz); ent_sgn.push_back(sg);
        tmpR.push_back(p); tmpR.push_back(q);
      };
      while (inz < Ajc[j + 1] && Air[inz] < bs + span) {
        long long idx = Air[inz] - bs;
        const bool imag = idx >= (long long)nr * nr;
        if (imag) idx -= (long long)nr * nr;
        int p = (int)(idx % nr), q = (int)(idx / nr);
        if (!cplx) add_entry(p, q, 1.0);
        else if (!imag) {                              // Re part a at (p,q): E has a at (p,q) and (p+n,q+n)
          add_entry(p, q, 1.0); add_entry(p + nr, q + nr, 1.0);
        } else {                                       // Im part b at (p>q): E has +b at (p+n,q), -b at (q+n,p)  (+ mirrors)
          SB_CHECK(p != q, "getada3: imaginary diagonal entry in Hermitian block %d", k);
          add_entry(std::max(p, q) + nr, std::min(p, q), 1.0); add_entry(std::min(p, q) + nr, std::max(p, q), -1.0);
        }
        inz++;
      }
      P.e1 = (int)ent_p.size();
      std::sort(tmpR.begin(), tmpR.end());
      tmpR.erase(std::unique(tmpR.begin(), tmpR.end()), tmpR.end());
      // Rlist / tt_ptr carry one extra slot per pair so that tt_ptr[r0 + rho + 1] is always valid
      P.r0 = (int)Rlist.size(); P.r = (int)tmpR.size();
      for (int v : tmpR) Rlist.push_back(v);
      Rlist.push_back(-1);
      percol.assign(tmpR.size(), {});
      for (int e = P.e0; e < P.e1; e++) {
        const int pp = ent_p[e], qq = ent_q[e];
        const int rp = (int)(std::lower_bound(tmpR.begin(), tmpR.end(), pp) - tmpR.begin());
        const int rq = (int)(std::lower_bound(tmpR.begin(), tmpR.end(), qq) - tmpR.begin());
        ent_lin.push_back(std::max(pp, qq) + std::min(pp, qq) * n);
        if (pp == qq) percol[rp].push_back({pp, {ent_src[e], ent_sgn[e]}});
        else {                                      // sym(X) = (X+X')/2   (spscale.c:227-229)
          percol[rq].push_back({pp, {ent_src[e], 0.5 * ent_sgn[e]}});
          percol[rp].push_back({qq, {ent_src[e], 0.5 * ent_sgn[e]}});
        }
      }
      for (size_t rho = 0; rho < tmpR.size(); rho++) {
        tt_ptr.push_back((int)tt_col.size());
        for (auto &t : percol[rho]) { tt_col.push_back(t.first); tt_row.push_back(tmpR[rho]); tt_src.push_back(t.second.first); tt_w.push_back(t.second.second); }
      }
      tt_ptr.push_back((int)tt_col.size());
      pl->pairs.push_back(P);
    }
  }
  pl->cpair_beg[m] = (int)pl->pairs.size();
  pl->n_tt = (long long)tt_col.size();
  // ---- union pattern U_k per block; blocks that use less than a quarter of their lower triangle
  // evaluate W only there ("sparse mode"), and their entries index into U_k instead of the n x n array
  std::vector<std::vector<int>> ulin(nblk);
  for (auto &P : pl->pairs)
    for (int e = P.e0; e < P.e1; e++) ulin[P.k].push_back(ent_lin[e]);
  std::vector<int> ublk_off(nblk + 1, 0), u_p, u_q;
  pl->blk_sparse.assign(nblk, 0);
  for (sb_idx k = 0; k < nblk; k++) {
    auto &v = ulin[k];
    std::sort(v.begin(), v.end());
    v.erase(std::unique(v.begin(), v.end()), v.end());
    const long long n = pl->blk_n[k];
    pl->blk_sparse[k] = ((long long)v.size() * 8 <= n * (n + 1));
    ublk_off[k] = (int)u_p.size();
    if (pl->blk_sparse[k]) {
      for (int lin : v) { u_p.push_back((int)(lin % n)); u_q.push_back((int)(lin / n)); }
      pl->max_nu = std::max(pl->max_nu, (int)v.size());
    }
  }
  ublk_off[nblk] = (int)u_p.size();
  for (auto &P : pl->pairs) {
    P.sparse = pl->blk_sparse[P.k];
    if (P.sparse) {
      const auto &v = ulin[P.k];
      for (int e = P.e0; e < P.e1; e++) ent_lin[e] = (int)(std::lower_bound(v.begin(), v.end(), ent_lin[e]) - v.begin());
    }
  }
  // ---- shared-memory staging of W in the dots kernel: packed index per entry, partner lists per block
  std::vector<int> ent_pk(ent_lin.size());
  std::vector<int> blkp_beg(nblk + 1, 0);
  for (auto &P : pl->pairs) blkp_beg[P.k + 1]++;
  for (sb_idx k = 0; k < nblk; k++) blkp_beg[k + 1] += blkp_beg[k];
  std::vector<BlkPartner> blkp(pl->pairs.size());
  std::vector<int> blkp_pair(pl->pairs.size());        // pair index of every list entry
  {
    // the partner list of a block, sparsest constraint first (ties: constraint number): a pair's partners in the
    // fused path are the entries up to and including its own position
    std::vector<std::vector<int>> byblk(nblk);
    for (size_t pi = 0; pi < pl->pairs.size(); pi++) byblk[pl->pairs[pi].k].push_back((int)pi);
    for (sb_idx k = 0; k < nblk; k++) {
      auto &v = byblk[k];
      std::stable_sort(v.begin(), v.end(), [&](int a, int b) {
        const int ea = pl->pairs[a].e1 - pl->pairs[a].e0, eb = pl->pairs[b].e1 - pl->pairs[b].e0;
        return ea != eb ? ea < eb : pl->pairs[a].j < pl->pairs[b].j;
      });
      for (size_t t = 0; t < v.size(); t++) {
        AdaPair &P = pl->pairs[v[t]];
        P.rank = (int)t;
        blkp[blkp_beg[k] + t] = BlkPartner{P.j, P.e0, P.e1, ent_src[P.e0]};
        blkp_pair[blkp_beg[k] + t] = v[t];
      }
    }
    for (auto &P : pl->pairs) {
      const long long n = pl->blk_n[P.k];
      for (int e = P.e0; e < P.e1; e++) {
        if (P.sparse) ent_pk[e] = ent_lin[e];
        else { const long long pp = ent_lin[e] % n, qq = ent_lin[e] / n; ent_pk[e] = (int)((qq * (2 * n - qq + 1)) / 2 - qq + pp); }
      }
    }
  }
  pl->use_map = (m <= 10000);          // row -> slot map of one ADA column in shared memory (<= 40 KB)
  {
    const long long mapb = pl->use_map ? (((long long)m * 4 + 7) & ~7LL) : 0;
    const long long cap = (220 * 1024 - mapb) / 8;
    long long wc = 1;
    for (sb_idx k = 0; k < nblk; k++) {
      if (blkp_beg[k + 1] == blkp_beg[k]) continue;
      const long long n = pl->blk_n[k];
      const long long wsz = pl->blk_sparse[k] ? (ublk_off[k + 1] - ublk_off[k]) : n * (n + 1) / 2;
      if (wsz <= cap) wc = std::max(wc, wsz);
    }
    pl->wcap = (int)wc;
    pl->dots_smem = (size_t)(wc * 8 + mapb);
    const double avg = pl->pairs.empty() ? 0.0 : (double)ent_lin.size() / (double)pl->pairs.size();
    pl->dots_group = avg <= 6.0 ? 4 : (avg <= 12.0 ? 8 : (avg <= 24.0 ? 16 : 32));
    std::vector<double> bent(nblk, 0.0), bcnt(nblk, 0.0);
    for (auto &P : pl->pairs) { bent[P.k] += P.e1 - P.e0; bcnt[P.k] += 1.0; }
    std::vector<int> bgrp(std::max<sb_idx>(nblk, 1), 32);
    for (sb_idx k = 0; k < nblk; k++) {
      const double a2 = bcnt[k] > 0 ? bent[k] / bcnt[k] : 0.0;
      bgrp[k] = a2 <= 6.0 ? 4 : (a2 <= 12.0 ? 8 : (a2 <= 24.0 ? 16 : 32));
    }
    SB_TRY(pl->d_blk_group.upload(bgrp));
  }
  // ---- batches of whole constraints, workspace bounded
  const long long BUDGET = (long long)96 << 20;     // doubles (768 MB)
  std::vector<GemmDesc> descs(pl->pairs.size());
  std::vector<GemmTile> tiles;
  int c = 0;
  while (c < m) {
    sb200_ada_plan::Batch B{}; B.c0 = c; B.p0 = pl->cpair_beg[c]; B.tile0 = (int)tiles.size();
    long long ws = 0;
    while (c < m) {
      long long need = 0;
      for (int p = pl->cpair_beg[c]; p < pl->cpair_beg[c + 1]; p++) {
        long long n = pl->blk_n[pl->pairs[p].k];
        const long long wsz = pl->pairs[p].sparse ? (ublk_off[pl->pairs[p].k + 1] - ublk_off[pl->pairs[p].k]) : n * n;
        need += wsz + n * pl->pairs[p].r;
        if (pl->cpair_beg[c + 1] - pl->cpair_beg[c] > 1) need += blkp_beg[pl->pairs[p].k + 1] - blkp_beg[pl->pairs[p].k] + 1;
      }
      if (ws > 0 && ws + need > BUDGET) break;
      for (int p = pl->cpair_beg[c]; p < pl->cpair_beg[c + 1]; p++) {
        AdaPair &P = pl->pairs[p];
        long long n = pl->blk_n[P.k];
        P.tt_off = ws; ws += n * P.r;
        P.w_off = ws; ws += P.sparse ? (ublk_off[P.k + 1] - ublk_off[P.k]) : n * n;
        P.part_off = ws;
        if (pl->cpair_beg[c + 1] - pl->cpair_beg[c] > 1) { ws += blkp_beg[P.k + 1] - blkp_beg[P.k] + 1; B.nmulti++; }
        if (P.sparse) { B.nsparse++; continue; }
        GemmDesc g{};
        g.offA = pl->blk_off[P.k]; g.gatherOff = P.r0; g.lda = (int)n; g.a_tri = TRI_NONE;
        g.offB = P.tt_off; g.ldb = (int)n; g.b_tri = TRI_NONE;
        g.offC = P.w_off; g.ldc = (int)n; g.M = g.N = (int)n; g.K = P.r; g.lower = 1; g.accumulate = 0; g.alpha = 1.0;
        descs[p] = g;
        gemm_add_tiles(tiles, p, (int)n, (int)n, true);
      }
      c++;
    }
    B.c1 = c; B.p1 = pl->cpair_beg[c]; B.ws = ws; B.ntiles = (int)tiles.size() - B.tile0;
    pl->ws_max = std::max(pl->ws_max, ws);
    pl->batches.push_back(B);
  }
  {
    long long nnz_lq = 0;
    for (sb_idx j = 0; j < m; j++) nnz_lq += (nblk ? Ajc1[j] : Ajc[j + 1]) - Ajc[j];
    pl->lq_dense = pl->lq_rows >= 64 && nnz_lq >= 32 * (long long)m && nnz_lq * 5 > pl->lq_rows * (long long)m &&
                   pl->lq_rows * (long long)m <= ((long long)64 << 20);
  }
  // ---- pattern of DAt.q: per column the Lorentz cones it touches (trace row and/or norm-bound rows)
  if (nq > 0) {
    std::vector<long long> qjc(m + 1, 0), qlo, qhi;
    std::vector<int> qir, qts;
    const long long tr0 = lpN, nb0 = qstart[0], nb1 = qstart[nq];
    long long seglen = 0;
    for (sb_idx j = 0; j < m; j++) {
      qjc[j] = (long long)qir.size();
      sb_idx p = Ajc[j];
      const sb_idx pend = nblk ? Ajc1[j] : Ajc[j + 1];
      while (p < pend && Air[p] < tr0) p++;
      sb_idx pt = p;                                   // trace entries [pt, pn)
      while (p < pend && Air[p] < tr0 + nq) p++;
      sb_idx pn = p;                                   // norm-bound entries [pn, pe)
      while (p < pend && Air[p] < nb1) p++;
      const sb_idx pe = p;
      SB_CHECK(pn == pe || Air[pn] >= nb0, "getDAtm: row %lld between the Lorentz trace and norm-bound parts", (long long)Air[pn]);
      sb_idx a = pt, b2 = pn;
      while (a < pn || b2 < pe) {
        const int ka = a < pn ? (int)(Air[a] - tr0) : 0x7fffffff;
        int kb = 0x7fffffff;
        if (b2 < pe) kb = (int)(std::upper_bound(qstart, qstart + nq + 1, Air[b2]) - qstart) - 1;
        const int kk = std::min(ka, kb);
        qir.push_back(kk);
        qts.push_back(ka == kk ? (int)a : -1);
        if (ka == kk) a++;
        long long l0 = b2;
        if (kb == kk) while (b2 < pe && Air[b2] < qstart[kk + 1]) b2++;
        qlo.push_back(l0); qhi.push_back(b2);
        seglen += b2 - l0;
      }
    }
    qjc[m] = (long long)qir.size();
    pl->dq_nnz = (long long)qir.size();
    pl->dq_wide = pl->dq_nnz > 0 && seglen / pl->dq_nnz >= 16;
    SB_TRY(pl->d_dq_jc.upload(qjc)); SB_TRY(pl->d_dq_ir.upload(qir)); SB_TRY(pl->d_dq_tsrc.upload(qts));
    SB_TRY(pl->d_dq_lo.upload(qlo)); SB_TRY(pl->d_dq_hi.upload(qhi));
    SB_TRY(pl->d_dq_pr.alloc((size_t)std::max<long long>(pl->dq_nnz, 1)));
  }
  // ---- upload
  std::vector<long long> v64;
  auto up64 = [&](DevBuf<long long> &d, const sb_idx *p, size_t n) { v64.assign(p, p + n); return d.upload(v64); };
  std::vector<int> v32;
  SB_TRY(up64(pl->d_Ajc, Ajc, m + 1));
  SB_TRY(up64(pl->d_Ajc1, Ajc1, m));
  SB_TRY(up64(pl->d_Ajcend, Ajc + 1, m));
  SB_TRY(up64(pl->d_adajc, adajc, m + 1));
  if (nq) SB_TRY(up64(pl->d_qstart, qstart, nq + 1)); else SB_TRY(pl->d_qstart.alloc(1));
  SB_TRY(to_i32(Air, (size_t)Ajc[m], v32, "At.ir")); SB_TRY(pl->d_Air.upload(v32));
  pl->h_Air = v32;
  SB_TRY(to_i32(adair, (size_t)adajc[m], v32, "ADA.ir")); SB_TRY(pl->d_adair.upload(v32));
  SB_TRY(pl->d_blk_n.upload(pl->blk_n)); SB_TRY(pl->d_blk_off.upload(pl->blk_off));
  SB_TRY(pl->d_cpair_beg.upload(pl->cpair_beg));
  SB_TRY(pl->d_ent_lin.upload(ent_lin)); SB_TRY(pl->d_ent_src.upload(ent_src));
  if (pl->herm) {
    // <E(A_i), E(W)> = 2 Re tr(A_i^H W): every embedded entry carries sign * 1/2 (real blocks of a mixed plan: 1)
    std::vector<double> sc(ent_sgn.size());
    for (auto &P : pl->pairs)
      for (int e = P.e0; e < P.e1; e++) sc[e] = ent_sgn[e] * (pl->blk_cplx[P.k] ? 0.5 : 1.0);
    SB_TRY(pl->d_ent_scale.upload(sc));
    SB_TRY(pl->d_blk_nraw.upload(pl->blk_nraw)); SB_TRY(pl->d_blk_cplx.upload(pl->blk_cplx)); SB_TRY(pl->d_blk_rawoff.upload(pl->blk_rawoff));
    SB_TRY(pl->d_De.alloc((size_t)std::max<long long>(pl->lenud_emb, 1)));
  }
  SB_TRY(pl->d_tt_ptr.upload(tt_ptr)); SB_TRY(pl->d_tt_col.upload(tt_col)); SB_TRY(pl->d_tt_src.upload(tt_src));
  SB_TRY(pl->d_tt_row.upload(tt_row));
  SB_TRY(pl->d_tt_w.upload(tt_w));
  SB_TRY(pl->d_ublk_off.upload(ublk_off)); SB_TRY(pl->d_u_p.upload(u_p)); SB_TRY(pl->d_u_q.upload(u_q));
  SB_TRY(pl->d_blkp_beg.upload(blkp_beg)); SB_TRY(pl->d_blkp.upload(blkp)); SB_TRY(pl->d_ent_pk.upload(ent_pk));
  SB_TRY(pl->d_Rlist.upload(Rlist));
  // ---- fused path: compact partial-sum workspace, scratch slot per resident CTA
  {
    bool ok = !pl->herm && !pl->pairs.empty() && !getenv("SB200_NO_FUSED_ADA3");
    int maxn = 0; long long max_tt = 1;
    for (auto &P : pl->pairs) {
      if (P.sparse || pl->blk_n[P.k] > FUSED_MAX_N) ok = false;
      maxn = std::max(maxn, pl->blk_n[P.k]);
      max_tt = std::max(max_tt, (long long)pl->blk_n[P.k] * (P.r + FKC - 1));   // T rows padded to whole k-slabs
    }
    long long fws = 0;
    for (sb_idx c2 = 0; c2 < m; c2++) {
      const bool multi = pl->cpair_beg[c2 + 1] - pl->cpair_beg[c2] > 1;
      for (int p = pl->cpair_beg[c2]; p < pl->cpair_beg[c2 + 1]; p++) {
        pl->pairs[p].fpart_off = fws;
        if (multi) { fws += blkp_beg[pl->pairs[p].k + 1] - blkp_beg[pl->pairs[p].k] + 1; pl->any_multi = 1; }
      }
    }
    pl->fused_ok = ok;
    if (ok) {
      const int nst = (maxn + 31) / 32, items = nst * (nst + 1) / 2;
      pl->fused_small = items <= 8;
      pl->fused_threads = pl->fused_small ? 256 : 512;
      // per block: lower supertiles sorted by their number of fragments (a round costs what its dearest item costs)
      std::vector<int> ibeg(nblk + 1, 0);
      std::vector<int2> its;
      for (sb_idx k = 0; k < nblk; k++) {
        ibeg[k] = (int)its.size();
        const int nk = pl->blk_n[k], nt = (nk + 7) / 8, ns = (nk + 31) / 32;
        std::vector<std::pair<int, int2>> v;
        for (int I = 0; I < ns; I++)
          for (int J = 0; J <= I; J++) {
            const int nra = std::min(4, nt - 4 * I), ncb = std::min(4, nt - 4 * J);
            int cost = 0;
            for (int a2 = 0; a2 < nra; a2++) for (int b2 = 0; b2 < ncb; b2++) if (I != J || a2 >= b2) cost++;
            v.push_back({-cost, make_int2(I, J)});
          }
        std::stable_sort(v.begin(), v.end(), [](const std::pair<int, int2> &x, const std::pair<int, int2> &y) { return x.first < y.first; });
        for (auto &e : v) its.push_back(e.second);
      }
      ibeg[nblk] = (int)its.size();
      SB_TRY(pl->d_fitem_beg.upload(ibeg)); SB_TRY(pl->d_fitems.upload(its));
      // evaluation mode of every pair: walk each block's list in order, keep the union of the patterns seen so far
      std::vector<int> need_pq;
      std::vector<char> seen;
      std::vector<double> cost(pl->pairs.size(), 0.0);
      long long ndense = 0;
      for (sb_idx k = 0; k < nblk; k++) {
        const long long nk = pl->blk_n[k], tri = nk * (nk + 1) / 2;
        seen.assign((size_t)tri, 0);
        std::vector<int> uni;                           // packed indices of the union, in order of first appearance
        for (int t = blkp_beg[k]; t < blkp_beg[k + 1]; t++) {
          AdaPair &P = pl->pairs[blkp_pair[t]];
          for (int e = P.e0; e < P.e1; e++) if (!seen[ent_pk[e]]) { seen[ent_pk[e]] = 1; uni.push_back(ent_pk[e]); }
          long long nfull = 0;                          // nonzeros of sym(A_jk)
          for (int rho = 0; rho < P.r; rho++) nfull += tt_ptr[P.r0 + rho + 1] - tt_ptr[P.r0 + rho];
          const long long nu = (long long)uni.size();
          if (nu * 16 <= tri && !getenv("SB200_ADA3_DENSE_ONLY")) {
            P.mode = (nfull <= 2 * nk) ? 2 : 1;
            P.need_off = (long long)need_pq.size(); P.need_cnt = (int)nu;
            for (int pk : uni) {                         // packed index -> (p, q): column q starts at q(2n-q+1)/2 - q
              long long q = 0;
              { long long lo = 0, hi = nk - 1; while (lo < hi) { long long mid = (lo + hi + 1) >> 1; if ((mid * (2 * nk - mid + 1)) / 2 <= pk) lo = mid; else hi = mid - 1; } q = lo; }
              const long long pp = pk - ((q * (2 * nk - q + 1)) / 2 - q);
              need_pq.push_back((int)(pp | (q << 16)));
            }
            cost[blkp_pair[t]] = (double)nu * (P.mode == 2 ? (double)nfull : (double)P.r) * 8.0 + (P.mode == 1 ? (double)nk * P.r * 4.0 : 0.0);
          } else {
            P.mode = 0; P.need_off = 0; P.need_cnt = 0; ndense++;
            cost[blkp_pair[t]] = (double)tri * P.r + (double)nk * P.r * 4.0;
          }
        }
      }
      pl->fused_ndense = ndense;
      {
        std::vector<int> slots;
        for (auto &P : pl->pairs) {
          P.slot_off = (long long)slots.size();
          const sb_idx *rb = adair + adajc[P.j], *re = adair + adajc[P.j + 1];
          const int tb = blkp_beg[P.k];
          for (int t = 0; t <= P.rank; t++) {
            const sb_idx want = blkp[tb + t].j;
            const sb_idx *it = std::lower_bound(rb, re, want);
            slots.push_back((it != re && *it == want) ? (int)(it - rb) : -1);
          }
        }
        if (slots.empty()) slots.push_back(-1);
        SB_TRY(pl->d_fslot.upload(slots));
      }
      // pairs are handed out most expensive first (dense products, then the entry-wise ones)
      std::vector<int> order(pl->pairs.size());
      for (size_t i = 0; i < order.size(); i++) order[i] = (int)i;
      // dense products first, then the entry-wise pairs; inside a class BLOCK BY BLOCK (then dearest first): the resident
      // CTAs then share two or three blocks' D_k and partner entries in L2.  Handing the pairs out by cost alone
      // interleaved all blocks (pair numbering follows the constraints): 91 MB of partner entries + 47 MB of T slots
      // + 20 MB of D for the 64 x 200 problem, far more than the 50 MB L2 of an H100.
      std::stable_sort(order.begin(), order.end(), [&](int a, int b) {
        const int ca = pl->pairs[a].mode != 0, cb = pl->pairs[b].mode != 0;
        if (ca != cb) return ca < cb;
        if (pl->pairs[a].k != pl->pairs[b].k) return pl->pairs[a].k < pl->pairs[b].k;
        return cost[a] > cost[b];
      });
      if (need_pq.empty()) need_pq.push_back(0);
      SB_TRY(pl->d_fneed.upload(need_pq)); SB_TRY(pl->d_forder.upload(order));
      // ---- strips: (pair, column strip) work items for blocks that leave no room for a second resident CTA
      if (!pl->fused_small && getenv("SB200_STRIP_ADA3")) {         // opt-in, parity-tested alternative to the whole-pair kernel (DESIGN.md)
        bool sok = true;
        std::vector<int> bgb(nblk + 1, 0);
        std::vector<StripGroup> groups;
        std::vector<int2> sitems;
        int gwmax = 0;
        for (sb_idx k = 0; k < nblk && sok; k++) {
          bgb[k] = (int)groups.size();
          const int nk = pl->blk_n[k], ns = (nk + 31) / 32, nt = (nk + 7) / 8;
          int J = 0;
          while (J < ns) {
            int J1 = J, nit = 0; long long ent = 0;
            while (J1 < ns) {
              long long e2 = 0;
              for (int cc = 32 * J1; cc < std::min(nk, 32 * J1 + 32); cc++) e2 += nk - cc;
              const int it = ns - J1;
              if (J1 > J && (ent + e2 > STRIP_WCAP || nit + it > 8)) break;
              ent += e2; nit += it; J1++;
            }
            if (ent > STRIP_WCAP) { sok = false; break; }
            StripGroup G{};
            G.c0 = 32 * J; G.c1 = std::min(nk, 32 * J1);
            G.base = (int)(((long long)G.c0 * (2 * nk - G.c0 + 1)) / 2);
            G.gw_al = (G.c1 - G.c0 + 1) & ~1;
            G.item_beg = (int)sitems.size();
            std::vector<std::pair<int, int2>> v;
            for (int Jc = J; Jc < J1; Jc++)
              for (int I = Jc; I < ns; I++) {
                const int nra = std::min(4, nt - 4 * I), ncb = std::min(4, nt - 4 * Jc);
                int cst = 0;
                for (int a2 = 0; a2 < nra; a2++) for (int b2 = 0; b2 < ncb; b2++) if (I != Jc || a2 >= b2) cst++;
                v.push_back({-cst, make_int2(I, Jc)});
              }
            std::stable_sort(v.begin(), v.end(), [](const std::pair<int, int2> &x, const std::pair<int, int2> &y) { return x.first < y.first; });
            for (auto &e : v) sitems.push_back(e.second);
            G.item_end = (int)sitems.size();
            gwmax = std::max(gwmax, G.c1 - G.c0);
            groups.push_back(G);
            J = J1;
          }
        }
        bgb[nblk] = (int)groups.size();
        if (sok) {
          auto group_of = [&](int k, int q) {                  // strip of column q in block k
            for (int g = bgb[k]; g < bgb[k + 1]; g++) if (q < groups[g].c1) return g - bgb[k];
            return bgb[k + 1] - bgb[k] - 1;
          };
          // entries of every partner, strip by strip (At order inside a strip)
          std::vector<int> feoff(nblk + 1, 0), fe_ptr, fe_src;
          std::vector<unsigned short> fe_pk;
          std::vector<int> lanes(std::max<sb_idx>(nblk, 1), 32);
          std::vector<std::vector<int>> bucket;
          for (sb_idx k = 0; k < nblk; k++) {
            feoff[k] = (int)fe_ptr.size();
            const int ng = bgb[k + 1] - bgb[k];
            const long long nk = pl->blk_n[k];
            const size_t ent0 = fe_pk.size();
            for (int t = blkp_beg[k]; t < blkp_beg[k + 1]; t++) {
              const AdaPair &P = pl->pairs[blkp_pair[t]];
              bucket.assign(ng, {});
              for (int e = P.e0; e < P.e1; e++) bucket[group_of((int)k, (int)(ent_lin[e] / nk))].push_back(e);
              for (int g = 0; g < ng; g++) {
                fe_ptr.push_back((int)fe_pk.size());
                for (int e : bucket[g]) {
                  const long long pp = ent_lin[e] % nk, qq = ent_lin[e] / nk;
                  fe_pk.push_back((unsigned short)((qq * (2 * nk - qq + 1)) / 2 - qq + pp - groups[bgb[k] + g].base));
                  fe_src.push_back(ent_src[e]);
                }
              }
            }
            const double cnt = (double)(blkp_beg[k + 1] - blkp_beg[k]) * ng;
            const double a2 = cnt > 0 ? (double)(fe_pk.size() - ent0) / cnt : 0.0;
            lanes[k] = a2 <= 6.0 ? 4 : (a2 <= 12.0 ? 8 : (a2 <= 24.0 ? 16 : 32));
          }
          feoff[nblk] = (int)fe_ptr.size();
          fe_ptr.push_back((int)fe_pk.size());
          // per (pair, strip): its share of the needed set, its partial-sum slot; the work list
          std::vector<int> pair_pg(pl->pairs.size() + 1, 0), sneed;
          std::vector<StripPG> pgs;
          std::vector<StripWork> work;
          std::vector<double> wcost;
          long long sws = 0, smax_tt = 2;
          for (size_t pi = 0; pi < pl->pairs.size(); pi++) {
            const AdaPair &P = pl->pairs[pi];
            const int k = P.k, ng = bgb[k + 1] - bgb[k];
            const long long nk = pl->blk_n[k];
            pair_pg[pi] = (int)pgs.size();
            bucket.assign(ng, {});
            if (P.mode != 0)
              for (int u = 0; u < P.need_cnt; u++) { const int v = need_pq[(size_t)P.need_off + u]; bucket[group_of(k, v >> 16)].push_back(v); }
            for (int g = 0; g < ng; g++) {
              const StripGroup &G = groups[bgb[k] + g];
              StripPG X{};
              X.need_beg = (int)sneed.size(); X.need_cnt = (int)bucket[g].size();
              for (int v : bucket[g]) sneed.push_back(v);
              if (P.mode != 0 && X.need_cnt == 0) { X.part_off = -1; pgs.push_back(X); continue; }
              X.part_off = sws; sws += P.rank + 2;
              pgs.push_back(X);
              double cst;
              if (P.mode == 0) {
                double fr = 0;
                const int nt = (int)((nk + 7) / 8);
                for (int it = G.item_beg; it < G.item_end; it++) {
                  const int I = sitems[it].x, Jc = sitems[it].y;
                  const int nra = std::min(4, nt - 4 * I), ncb = std::min(4, nt - 4 * Jc);
                  for (int a2 = 0; a2 < nra; a2++) for (int b2 = 0; b2 < ncb; b2++) if (I != Jc || a2 >= b2) fr += 1.0;
                }
                cst = fr * 64.0 * P.r + (double)(G.c1 - G.c0) * P.r * 4.0;
              } else {
                long long nfull = tt_ptr[P.r0 + P.r] - tt_ptr[P.r0];
                cst = (double)X.need_cnt * (P.mode == 2 ? (double)nfull : (double)P.r) * 8.0 + (P.mode == 1 ? (double)(G.c1 - G.c0) * P.r * 4.0 : 0.0);
              }
              work.push_back(StripWork{(int)pi, g}); wcost.push_back(cst);
              if (P.mode != 2) smax_tt = std::max(smax_tt, (long long)G.gw_al * P.r);
            }
          }
          pair_pg[pl->pairs.size()] = (int)pgs.size();
          std::vector<int> ord(work.size());
          for (size_t i = 0; i < ord.size(); i++) ord[i] = (int)i;
          std::stable_sort(ord.begin(), ord.end(), [&](int a, int b) { return wcost[a] > wcost[b]; });
          std::vector<StripWork> work2(work.size());
          for (size_t i = 0; i < ord.size(); i++) work2[i] = work[ord[i]];
          if (sneed.empty()) sneed.push_back(0);
          if (fe_src.empty()) { fe_src.push_back(0); fe_pk.push_back(0); }
          pl->strip_ldA = ((maxn + 7) & ~7) + 4;
          pl->strip_ldB = ((gwmax + 7) & ~7) + 4;
          pl->strip_smem = sizeof(double) * ((size_t)STRIP_WCAP + STRIP_STAGES * FKC * (size_t)(pl->strip_ldA + pl->strip_ldB));
          const int per_sm = (int)std::max<size_t>(1, std::min<size_t>(2, (226 * 1024) / (pl->strip_smem + 1024)));
          pl->strip_nwork = (int)work2.size();
          pl->strip_grid = (int)std::min<long long>((long long)work2.size(), (long long)ctx().sm_count * per_sm);
          pl->strip_scratch_stride = (smax_tt + 1) & ~1LL;
          pl->strip_nent = (long long)fe_src.size();
          if (pl->strip_nwork > 0 && per_sm >= 2) {
            SB_TRY(pl->d_sgroups.upload(groups)); SB_TRY(pl->d_spg.upload(pgs)); SB_TRY(pl->d_swork.upload(work2));
            SB_TRY(pl->d_sblk_grp_beg.upload(bgb)); SB_TRY(pl->d_spair_pg.upload(pair_pg)); SB_TRY(pl->d_sblk_feoff.upload(feoff));
            SB_TRY(pl->d_sfe_ptr.upload(fe_ptr)); SB_TRY(pl->d_sfe_src.upload(fe_src)); SB_TRY(pl->d_sfe_pk.upload(fe_pk));
            SB_TRY(pl->d_sneed.upload(sneed)); SB_TRY(pl->d_sblk_lanes.upload(lanes)); SB_TRY(pl->d_sitems.upload(sitems));
            SB_TRY(pl->d_sfe_val.alloc((size_t)pl->strip_nent));
            SB_TRY(pl->d_sscratch.alloc((size_t)(pl->strip_scratch_stride * std::max(pl->strip_grid, 1))));
            SB_TRY(pl->d_sws.alloc((size_t)std::max<long long>(sws, 1)));
            pl->strip_ok = true;
          }
        }
      }
      pl->fused_wcap = (maxn * (maxn + 1) / 2 + 1) & ~1;
      pl->fused_ldmax = ((maxn + 7) & ~7) + 4;
      pl->fused_smem = sizeof(double) * ((size_t)pl->fused_wcap + 4 * FKC * pl->fused_ldmax);
      const int per_sm = pl->fused_small ? (int)std::max<size_t>(1, std::min<size_t>(3, (200 * 1024) / pl->fused_smem)) : 1;
      pl->fused_grid = (int)std::min<long long>((long long)pl->pairs.size(), (long long)ctx().sm_count * per_sm);
      pl->fused_scratch_stride = (max_tt + 1) & ~1LL;
      pl->fws = fws;
      SB_TRY(pl->d_tt_val.alloc((size_t)std::max<long long>(pl->n_tt, 1)));
      SB_TRY(pl->d_fscratch.alloc((size_t)(pl->fused_scratch_stride * pl->fused_grid)));
      SB_TRY(pl->d_fws.alloc((size_t)std::max<long long>(fws, 1)));
      SB_TRY(pl->d_fcounter.alloc(1));
    }
  }
  SB_TRY(pl->d_pairs.upload(pl->pairs));
  SB_TRY(pl->d_descs.upload(descs)); SB_TRY(pl->d_tiles.upload(tiles));
  SB_TRY(pl->d_Atpr.alloc((size_t)std::max<long long>(pl->nnzA, 1)));
  SB_TRY(pl->d_dsqr.alloc((size_t)std::max<long long>(pl->lq_rows, 1)));
  SB_TRY(pl->d_ws.alloc((size_t)std::max<long long>(pl->ws_max, 1)));
  SB_TRY(pl->d_invperm.alloc((size_t)std::max(pl->m, 1)));
  v32.resize(m); for (int i = 0; i < m; i++) v32[i] = i;
  SB_TRY(pl->d_ident.upload(v32));
  SB_CUDA(cudaStreamSynchronize(ctx().stream));
  return 0;
}

extern "C" {

// Structure of the constraint matrix and of ADA.  All index arrays 0-based.
//   Ajc1[j]      absolute offset in At.ir of the first PSD nonzero of column j (= Ablkjc(:,3)),
//                which is also the end of its LP/Lorentz part
//   lpN          K.l ; nq = |K.q| ; qstart[0..nq]: first norm-bound row of each Lorentz cone (+ end)
//   blkstart/blkn first row and order of each (real) PSD block
int sb200_ada_plan_get(sb200_ada_plan **plan, sb_idx N, sb_idx m, const sb_idx *Ajc, const sb_idx *Air,
                       const sb_idx *Ajc1, sb_idx lpN, sb_idx nq, const sb_idx *qstart, sb_idx nblk,
                       const sb_idx *blkstart, const sb_idx *blkn, const sb_idx *adajc, const sb_idx *adair) {
  return sb200_ada_plan_get_h(plan, N, m, Ajc, Air, Ajc1, lpN, nq, qstart, nblk, nblk, blkstart, blkn, adajc, adair);
}
// Same with Hermitian PSD blocks: blocks [nreal, nblk) are Hermitian, rows [vec Re (lower triangle); vec Im (strictly
// lower)] = 2 n^2 rows each (pretransfo.m:456-480), udsqr [vec Re D; vec Im D] (spscale.c:332-435 spcpxdxd).
int sb200_ada_plan_get_h(sb200_ada_plan **plan, sb_idx N, sb_idx m, const sb_idx *Ajc, const sb_idx *Air,
                         const sb_idx *Ajc1, sb_idx lpN, sb_idx nq, const sb_idx *qstart, sb_idx nblk, sb_idx nreal,
                         const sb_idx *blkstart, const sb_idx *blkn, const sb_idx *adajc, const sb_idx *adair) {
  SB_TRY(ensure_init());
  SB_CHECK(nreal >= 0 && nreal <= nblk, "number of real PSD blocks out of range");
  Hash128 h = fnv1a(&N, sizeof N); h = fnv1a(&m, sizeof m, h);
  h = fnv1a(Ajc, sizeof(sb_idx) * (m + 1), h); h = fnv1a(Air, sizeof(sb_idx) * Ajc[m], h);
  h = fnv1a(Ajc1, sizeof(sb_idx) * m, h); h = fnv1a(&lpN, sizeof lpN, h); h = fnv1a(&nq, sizeof nq, h);
  if (nq) h = fnv1a(qstart, sizeof(sb_idx) * (nq + 1), h);
  h = fnv1a(&nblk, sizeof nblk, h); h = fnv1a(&nreal, sizeof nreal, h);
  if (nblk) { h = fnv1a(blkstart, sizeof(sb_idx) * nblk, h); h = fnv1a(blkn, sizeof(sb_idx) * nblk, h); }
  h = fnv1a(adajc, sizeof(sb_idx) * (m + 1), h); h = fnv1a(adair, sizeof(sb_idx) * adajc[m], h);
  auto it = g_ada_plans.find(h);
  if (it != g_ada_plans.end()) { it->second->cache_stamp = ++g_ada_clock; *plan = it->second; return 0; }
  sb200_ada_plan *pl = new sb200_ada_plan();
  int rc = ada_build(pl, N, m, Ajc, Air, Ajc1, lpN, nq, qstart, nblk, nreal, blkstart, blkn, adajc, adair);
  if (rc) { delete pl; return rc; }
  pl->key = h;
  // bounded cache: evict the least-recently-used plan that no device-resident owner has pinned (a HotPath, and the
  // CUDA graphs it captured, keep using a plan's device buffers for their whole lifetime)
  for (;;) {
    size_t unpinned = 0;
    auto lru = g_ada_plans.end();
    for (auto i2 = g_ada_plans.begin(); i2 != g_ada_plans.end(); ++i2) {
      if (i2->second->pins > 0) continue;
      unpinned++;
      if (lru == g_ada_plans.end() || i2->second->cache_stamp < lru->second->cache_stamp) lru = i2;
    }
    if (unpinned < 8) break;
    cudaStreamSynchronize(ctx().stream);
    delete lru->second;
    g_ada_plans.erase(lru);
  }
  pl->cache_stamp = ++g_ada_clock;
  g_ada_plans[h] = pl;
  *plan = pl;
  return 0;
}

// Values of At (host) -> device copy held by the plan (skipped when unchanged).
int sb200_ada_set_At_values(sb200_ada_plan *pl, const double *Atpr) {
  Hash128 h = fnv1a(Atpr, sizeof(double) * pl->nnzA);
  if (pl->have_vals && h == pl->val_hash) return 0;
  SB_CUDA(cudaMemcpyAsync(pl->d_Atpr.p, Atpr, sizeof(double) * pl->nnzA, cudaMemcpyHostToDevice, ctx().stream));
  SB_CUDA(cudaStreamSynchronize(ctx().stream));
  pl->val_hash = h; pl->have_vals = true; pl->lq_dense_valid = false; pl->tt_val_valid = false;
  return 0;
}
sb_idx sb200_ada_plan_nnz(const sb200_ada_plan *pl) { return pl->nnzADA; }
// Device arrays of At (CSC as given, and a CSR view built on first use) for the matrix-vector products of pcg.cu.
int sb200_ada_plan_csr(sb200_ada_plan *pl, const long long **Ajc, const int **Air, const double **Apr, const long long **rowptr,
                       const int **rowcol, const int **rowsrc, sb_idx *N, sb_idx *m, sb_idx *lpN, sb_idx *nq) {
  if (!pl->csr_built) {
    SB_CHECK(!ctx().capturing, "At's row-wise view must be built before graph capture (call once outside)");
    const long long N2 = pl->N; const int m2 = pl->m;
    std::vector<long long> rp((size_t)N2 + 1, 0);
    for (long long p = 0; p < pl->nnzA; p++) rp[pl->h_Air[p] + 1]++;
    for (long long r = 0; r < N2; r++) rp[r + 1] += rp[r];
    std::vector<int> rc((size_t)std::max<long long>(pl->nnzA, 1)), rs((size_t)std::max<long long>(pl->nnzA, 1));
    std::vector<long long> fill(rp.begin(), rp.end() - 1);
    for (int j = 0; j < m2; j++)
      for (long long p = pl->h_Ajc[j]; p < pl->h_Ajc[j + 1]; p++) { const long long t = fill[pl->h_Air[p]]++; rc[t] = j; rs[t] = (int)p; }
    SB_TRY(pl->d_rowptr.upload(rp)); SB_TRY(pl->d_rowcol.upload(rc)); SB_TRY(pl->d_rowsrc.upload(rs));
    SB_CUDA(cudaStreamSynchronize(ctx().stream));
    pl->csr_built = true;
  }
  *Ajc = pl->d_Ajc.p; *Air = pl->d_Air.p; *Apr = pl->d_Atpr.p; *rowptr = pl->d_rowptr.p; *rowcol = pl->d_rowcol.p; *rowsrc = pl->d_rowsrc.p;
  *N = pl->N; *m = pl->m; *lpN = pl->lpN; *nq = pl->nq;
  return 0;
}
// Diagnostics: per-phase cycle counts of the fused getada3 kernel (thread 0 of every CTA, summed over CTAs and launches
// since the call that enabled them): out[0..4] = prologue, T, dense product, entry-wise W, inner products; out[5..6] =
// dense / entry-wise pairs processed; out[7..10] = dense product split: wait for a slab, issue of the next slab's copies,
// DMMAs, accumulator write-back.  enable = 1 switches the counters on (and zeroes them), 0 reads them.  The kernel only
// carries the counters when the library is built with `make FUSED_PROF=1` (they cost 22 registers); otherwise zeros.
int sb200_ada_fused_profile(sb200_ada_plan *pl, int enable, unsigned long long *out) {
  if (enable) {
    if (!pl->d_fprof.p) SB_TRY(pl->d_fprof.alloc(16));
    SB_CUDA(cudaMemsetAsync(pl->d_fprof.p, 0, 16 * sizeof(unsigned long long), ctx().stream));
    pl->fprof_on = true;
    return 0;
  }
  SB_CHECK(pl->fprof_on, "fused profile counters were not enabled");
  SB_CUDA(cudaMemcpyAsync(out, pl->d_fprof.p, 16 * sizeof(unsigned long long), cudaMemcpyDeviceToHost, ctx().stream));
  SB_CUDA(cudaStreamSynchronize(ctx().stream));
  return 0;
}
// Ownership for device-resident callers: a retained plan is exempt from cache eviction until released.
int sb200_ada_plan_retain(sb200_ada_plan *pl) { if (pl) pl->pins++; return 0; }
int sb200_ada_plan_release(sb200_ada_plan *pl) { if (pl && pl->pins > 0) pl->pins--; return 0; }

static int set_invperm(sb200_ada_plan *pl, const sb_idx *perm, const int **out) {
  if (!perm) { *out = pl->d_ident.p; return 0; }
  std::vector<int> inv(pl->m);
  for (int i = 0; i < pl->m; i++) {
    SB_CHECK(perm[i] >= 0 && perm[i] < pl->m, "ordering permutation out of range");
    inv[perm[i]] = i;
  }
  SB_CUDA(cudaMemcpyAsync(pl->d_invperm.p, inv.data(), sizeof(int) * pl->m, cudaMemcpyHostToDevice, ctx().stream));
  SB_CUDA(cudaStreamSynchronize(ctx().stream));
  *out = pl->d_invperm.p;
  return 0;
}

// out = (accumulate ? in : 0) + Bd W Bd' on the ADA pattern (entries with invperm[i] <= invperm[c]), Bd m x R dense.
static int ata_dense(sb200_ada_plan *pl, const double *Bd, long long R, const double *w_dev, const int *invperm,
                     const double *in, double *out, int accumulate) {
  cudaStream_t st = ctx().stream;
  const int m = pl->m;
  auto it = pl->dense_sets.find(R);
  sb200_ada_plan::DenseSet *ds;
  if (it == pl->dense_sets.end()) {
    ds = new sb200_ada_plan::DenseSet();
    ds->R = R;
    const long long KC = 256;
    const long long cap = std::max<long long>(1, ((long long)32 << 20) / ((long long)m * m));
    ds->nchunk = (int)std::max<long long>(1, std::min((R + KC - 1) / KC, cap));
    const long long kc = (((R + ds->nchunk - 1) / ds->nchunk) + GK - 1) / GK * GK;
    ds->nchunk = (int)((R + kc - 1) / kc);
    std::vector<GemmDesc> descs; std::vector<GemmTile> tiles;
    for (int p = 0; p < ds->nchunk; p++) {
      GemmDesc g{};
      g.gatherOff = -1; g.alpha = 1.0; g.lda = g.ldb = g.ldc = m; g.a_tri = g.b_tri = TRI_NONE;
      g.offA = g.offB = (long long)p * kc * m; g.offC = (long long)p * m * m;
      g.M = g.N = m; g.K = (int)std::min<long long>(kc, R - (long long)p * kc); g.lower = 0; g.accumulate = 0;
      descs.push_back(g);
      gemm_add_tiles(tiles, p, m, m, false);
    }
    ds->ntiles = (int)tiles.size();
    SB_TRY(ds->descs.upload(descs)); SB_TRY(ds->tiles.upload(tiles));
    SB_CUDA(cudaStreamSynchronize(st));
    pl->dense_sets[R] = ds;
  } else ds = it->second;
  const long long tot = (long long)m * R;
  if (tot > pl->cap_Bd) { SB_TRY(pl->d_Bw.alloc((size_t)tot)); pl->cap_Bd = tot; }
  const long long ctot = (long long)ds->nchunk * m * m;
  if (ctot > pl->cap_Cp) { SB_TRY(pl->d_Cp.alloc((size_t)ctot)); pl->cap_Cp = ctot; }
  const double *Bw = Bd;
  if (w_dev) {
    scale_cols_kernel<<<(unsigned)std::min<long long>((tot + 255) / 256, 4096), 256, 0, st>>>(tot, m, w_dev, Bd, pl->d_Bw.p);
    SB_LAUNCH_CHECK_N("scale_cols_kernel");
    Bw = pl->d_Bw.p;
  }
  gemm_nt_launch(ds->ntiles, ctx().sm_count, st, ds->descs.p, ds->tiles.p, Bd, Bw, pl->d_Cp.p, nullptr);
  SB_LAUNCH_CHECK_N("gemm_nt_kernel");
  gather_dense_kernel<<<m, 256, 0, st>>>(m, pl->d_adajc.p, pl->d_adair.p, invperm, pl->d_Cp.p, ds->nchunk, in, out, accumulate);
  SB_LAUNCH_CHECK_N("gather_dense_kernel");
  return 0;
}
static int densify(sb200_ada_plan *pl, const long long *lo, const long long *hi, const int *ir, const double *pr, long long r0,
                   long long R, DevBuf<double> &dst) {
  cudaStream_t st = ctx().stream;
  const long long tot = (long long)pl->m * R;
  if ((long long)dst.n < tot) SB_TRY(dst.alloc((size_t)tot));
  SB_CUDA(cudaMemsetAsync(dst.p, 0, sizeof(double) * tot, st));
  dense_from_csc_kernel<<<pl->m, 256, 0, st>>>(pl->m, lo, hi, ir, pr, r0, R, dst.p);
  SB_LAUNCH_CHECK_N("dense_from_csc_kernel");
  return 0;
}

// getada1 on device values.  invperm_dev NULL = natural order (entries with i <= j).
int sb200_getada1_dev(sb200_ada_plan *pl, const double *dl_dev, const double *ddet_dev, const int *invperm_dev,
                      double *ada_out_dev) {
  SB_TRY(ensure_init());
  if (pl->m == 0) return 0;
  cudaStream_t st = ctx().stream;
  if (pl->lq_rows > 0) {
    dsqr_kernel<<<(unsigned)std::min<long long>((pl->lq_rows + 255) / 256, 2048), 256, 0, st>>>(
        pl->lpN, pl->nq, pl->d_qstart.p, dl_dev, ddet_dev, pl->d_dsqr.p);
    SB_LAUNCH_CHECK_N("dsqr_kernel");
  }
  if (pl->lq_dense) {
    if (!pl->lq_dense_valid) {
      SB_TRY(densify(pl, pl->d_Ajc.p, pl->d_Ajc1.p, pl->d_Air.p, pl->d_Atpr.p, 0, pl->lq_rows, pl->d_Bd_lq));
      pl->lq_dense_valid = true;
    }
    return ata_dense(pl, pl->d_Bd_lq.p, pl->lq_rows, pl->d_dsqr.p, invperm_dev ? invperm_dev : pl->d_ident.p, nullptr, ada_out_dev, 0);
  }
  ata_pattern_kernel<<<pl->m, 256, 0, st>>>(pl->m, pl->d_adajc.p, pl->d_adair.p, pl->d_Ajc.p, pl->d_Ajc1.p, pl->d_Air.p,
                                            pl->d_Atpr.p, pl->d_dsqr.p, invperm_dev ? invperm_dev : pl->d_ident.p,
                                            nullptr, ada_out_dev, 0, 1);
  SB_LAUNCH_CHECK_N("ata_pattern_kernel");
  return 0;
}

// getDAtm on the device: DAt.q values into the plan's own CSC (pattern fixed by At); q2 is d.q2, the
// concatenated norm-bound parts.  sb200_ada_plan_datq hands the device arrays out (for getada2_dev).
int sb200_getdatm_dev(sb200_ada_plan *pl, const double *q1_dev, const double *q2_dev) {
  SB_TRY(ensure_init());
  if (pl->nq == 0 || pl->dq_nnz == 0) return 0;
  const long long n = pl->dq_nnz;
  const long long q2row0 = pl->lpN + pl->nq;
  if (pl->dq_wide)
    datq_kernel<true><<<(unsigned)((n * 32 + 255) / 256), 256, 0, ctx().stream>>>(n, pl->d_dq_ir.p, pl->d_dq_tsrc.p, pl->d_dq_lo.p, pl->d_dq_hi.p,
        pl->d_Air.p, pl->d_Atpr.p, q1_dev, q2_dev, q2row0, pl->d_dq_pr.p);
  else
    datq_kernel<false><<<(unsigned)((n + 255) / 256), 256, 0, ctx().stream>>>(n, pl->d_dq_ir.p, pl->d_dq_tsrc.p, pl->d_dq_lo.p, pl->d_dq_hi.p,
        pl->d_Air.p, pl->d_Atpr.p, q1_dev, q2_dev, q2row0, pl->d_dq_pr.p);
  SB_LAUNCH_CHECK_N("datq_kernel");
  return 0;
}
int sb200_ada_plan_datq(sb200_ada_plan *pl, const long long **jc_dev, const int **ir_dev, const double **pr_dev, sb_idx *nnz) {
  *jc_dev = pl->d_dq_jc.p; *ir_dev = pl->d_dq_ir.p; *pr_dev = pl->d_dq_pr.p; *nnz = pl->dq_nnz;
  return 0;
}

// getada2 on device values: ada_out = ada_in + Q'Q (upper in perm order), Q = DAt.q as device CSC.
static int getada2_impl(sb200_ada_plan *pl, const long long *Qjc_dev, const int *Qir_dev, const double *Qpr_dev, long long nnzQ,
                        const int *invperm_dev, const double *ada_in_dev, double *ada_out_dev);
int sb200_getada2_dev(sb200_ada_plan *pl, const long long *Qjc_dev, const int *Qir_dev, const double *Qpr_dev,
                      const int *invperm_dev, const double *ada_in_dev, double *ada_out_dev) {
  // nnz(Q) is known when Q is the plan's own DAt.q (sb200_getdatm_dev); otherwise take the sparse route
  return getada2_impl(pl, Qjc_dev, Qir_dev, Qpr_dev, Qpr_dev == pl->d_dq_pr.p ? pl->dq_nnz : -1, invperm_dev, ada_in_dev, ada_out_dev);
}
static int getada2_impl(sb200_ada_plan *pl, const long long *Qjc_dev, const int *Qir_dev, const double *Qpr_dev, long long nnzQ,
                        const int *invperm_dev, const double *ada_in_dev, double *ada_out_dev) {
  SB_TRY(ensure_init());
  if (pl->m == 0) return 0;
  if (pl->nq >= 64 && nnzQ >= 32 * (long long)pl->m && nnzQ * 5 > (long long)pl->nq * pl->m && (long long)pl->nq * pl->m <= ((long long)64 << 20)) {
    SB_TRY(densify(pl, Qjc_dev, Qjc_dev + 1, Qir_dev, Qpr_dev, 0, pl->nq, pl->d_Bd));
    return ata_dense(pl, pl->d_Bd.p, pl->nq, nullptr, invperm_dev ? invperm_dev : pl->d_ident.p, ada_in_dev, ada_out_dev, 1);
  }
  ata_pattern_kernel<<<pl->m, 256, 0, ctx().stream>>>(pl->m, pl->d_adajc.p, pl->d_adair.p, Qjc_dev, Qjc_dev + 1, Qir_dev,
                                                       Qpr_dev, nullptr, invperm_dev ? invperm_dev : pl->d_ident.p,
                                                       ada_in_dev, ada_out_dev, 1, 1);
  SB_LAUNCH_CHECK_N("ata_pattern_kernel");
  return 0;
}

// getada3 on device values, in place on ada_dev.  first = number of leading constraints (in the
// order given by invperm) whose absd stays 0 (getada3.c:282-284); symmetrise = apply spmakesym.
int sb200_getada3_dev(sb200_ada_plan *pl, const double *udsqr_dev, const int *invperm_dev, sb_idx first,
                      double *ada_dev, double *absd_dev, int symmetrise) {
  SB_TRY(ensure_init());
  if (pl->m == 0) return 0;
  cudaStream_t st = ctx().stream;
  const int *ip = invperm_dev ? invperm_dev : pl->d_ident.p;
  // absd of the constraints with no PSD pair (diag(ADA) if there is no PSD cone at all, getada3.c:549-552)
  absd_nopsd_kernel<<<(pl->m + 255) / 256, 256, 0, st>>>(pl->m, pl->d_adajc.p, pl->d_adair.p, ip, (int)first,
                                                         pl->d_cpair_beg.p, ada_dev, absd_dev, pl->nblk == 0);
  SB_LAUNCH_CHECK_N("absd_nopsd_kernel");
  if (pl->herm) {
    int maxn = 0; for (int v : pl->blk_nraw) maxn = std::max(maxn, v);
    ada_embed_d_kernel<<<dim3((unsigned)std::min<long long>(((long long)maxn * maxn + 255) / 256, 1024), (unsigned)pl->nblk), 256, 0, st>>>(
        pl->d_blk_nraw.p, pl->d_blk_cplx.p, pl->d_blk_rawoff.p, pl->d_blk_off.p, udsqr_dev, pl->d_De.p);
    SB_LAUNCH_CHECK_N("ada_embed_d_kernel");
    udsqr_dev = pl->d_De.p;
  }
  if (pl->fused_ok) {
    const bool refresh_vals = !pl->tt_val_valid;
    if (!pl->tt_val_valid) {
      tt_val_kernel<<<(unsigned)std::min<long long>((pl->n_tt + 255) / 256, 2048), 256, 0, st>>>(pl->n_tt, pl->d_tt_w.p, pl->d_tt_src.p, pl->d_Atpr.p, pl->d_tt_val.p);
      SB_LAUNCH_CHECK_N("tt_val_kernel");
      if (!ctx().capturing) pl->tt_val_valid = true;      // inside a graph capture the launch must stay part of every replay
    }
    SB_CUDA(cudaMemsetAsync(pl->d_fcounter.p, 0, sizeof(int), st));
    if (pl->strip_ok) {
      if (refresh_vals) {
        gather_val_kernel<<<(unsigned)std::min<long long>((pl->strip_nent + 255) / 256, 2048), 256, 0, st>>>(pl->strip_nent, pl->d_sfe_src.p, pl->d_Atpr.p, pl->d_sfe_val.p);
        SB_LAUNCH_CHECK_N("gather_val_kernel");
      }
      StripArgs SA;
      SA.pairs = pl->d_pairs.p; SA.work = pl->d_swork.p; SA.nwork = pl->strip_nwork; SA.counter = pl->d_fcounter.p;
      SA.blk_n = pl->d_blk_n.p; SA.blk_off = pl->d_blk_off.p; SA.blk_grp_beg = pl->d_sblk_grp_beg.p; SA.groups = pl->d_sgroups.p; SA.items = pl->d_sitems.p;
      SA.pair_pg = pl->d_spair_pg.p; SA.pg = pl->d_spg.p;
      SA.tt_ptr = pl->d_tt_ptr.p; SA.tt_col = pl->d_tt_col.p; SA.tt_row = pl->d_tt_row.p; SA.tt_val = pl->d_tt_val.p; SA.Rlist = pl->d_Rlist.p; SA.udsqr = udsqr_dev;
      SA.scratch = pl->d_sscratch.p; SA.scratch_stride = pl->strip_scratch_stride;
      SA.blk_feoff = pl->d_sblk_feoff.p; SA.fe_ptr = pl->d_sfe_ptr.p; SA.fe_pk = pl->d_sfe_pk.p; SA.fe_val = pl->d_sfe_val.p;
      SA.need_pq = pl->d_sneed.p; SA.ws = pl->d_sws.p; SA.blk_lanes = pl->d_sblk_lanes.p; SA.ldA = pl->strip_ldA; SA.ldB = pl->strip_ldB;
      static bool sattr_done = false;
      if (!sattr_done) {
        SB_CUDA(cudaFuncSetAttribute(ada3_strip_kernel<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, 112 * 1024));
        sattr_done = true;
      }
      ada3_strip_kernel<2><<<pl->strip_grid, STRIP_THREADS, pl->strip_smem, st>>>(SA);
      SB_LAUNCH_CHECK_N("ada3_strip_kernel");
      ada3_strip_reduce_kernel<<<pl->m, 256, pl->use_map ? (size_t)pl->m * 4 : 0, st>>>(pl->d_adajc.p, pl->d_adair.p, ip, (int)first,
          pl->d_cpair_beg.p, pl->d_pairs.p, pl->d_blkp_beg.p, pl->d_blkp.p, pl->d_sblk_grp_beg.p, pl->d_spair_pg.p, pl->d_spg.p,
          pl->d_sws.p, ada_dev, absd_dev, pl->use_map, pl->m);
      SB_LAUNCH_CHECK_N("ada3_strip_reduce_kernel");
    } else {
    FusedArgs FA;
    FA.pairs = pl->d_pairs.p; FA.npairs = (int)pl->pairs.size(); FA.counter = pl->d_fcounter.p;
    FA.blk_n = pl->d_blk_n.p; FA.blk_off = pl->d_blk_off.p; FA.tt_ptr = pl->d_tt_ptr.p; FA.tt_col = pl->d_tt_col.p; FA.tt_row = pl->d_tt_row.p; FA.tt_val = pl->d_tt_val.p;
    FA.Rlist = pl->d_Rlist.p; FA.udsqr = udsqr_dev; FA.scratch = pl->d_fscratch.p; FA.scratch_stride = pl->fused_scratch_stride;
    FA.adajc = pl->d_adajc.p; FA.adair = pl->d_adair.p; FA.invperm = ip; FA.first = (int)first; FA.cpair_beg = pl->d_cpair_beg.p;
    FA.blkp_beg = pl->d_blkp_beg.p; FA.blkp = pl->d_blkp.p; FA.ent_pk = pl->d_ent_pk.p; FA.ent_src = pl->d_ent_src.p; FA.Atpr = pl->d_Atpr.p;
    FA.ws = pl->d_fws.p; FA.ada = ada_dev; FA.absd = absd_dev; FA.blk_group = pl->d_blk_group.p; FA.blk_item_beg = pl->d_fitem_beg.p; FA.items = pl->d_fitems.p; FA.need_pq = pl->d_fneed.p; FA.order = pl->d_forder.p; FA.wcap = pl->fused_wcap; FA.ldmax = pl->fused_ldmax; FA.prof = pl->fprof_on ? pl->d_fprof.p : nullptr; FA.slot = pl->d_fslot.p;
    static bool attr_done = false;
    if (!attr_done) {
      SB_CUDA(cudaFuncSetAttribute(ada3_fused_kernel<512, 1>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024 - 2048));   // + 1.7 KB static
      SB_CUDA(cudaFuncSetAttribute(ada3_fused_kernel<256, 2>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024 - 2048));
      attr_done = true;
    }
    if (pl->fused_small) ada3_fused_kernel<256, 2><<<pl->fused_grid, pl->fused_threads, pl->fused_smem, st>>>(FA);
    else ada3_fused_kernel<512, 1><<<pl->fused_grid, pl->fused_threads, pl->fused_smem, st>>>(FA);
    SB_LAUNCH_CHECK_N("ada3_fused_kernel");
    if (pl->any_multi) {
      ada3_reduce_kernel<<<pl->m, 256, pl->use_map ? (size_t)pl->m * 4 : 0, st>>>(0, pl->d_adajc.p, pl->d_adair.p, ip, (int)first,
          pl->d_cpair_beg.p, pl->d_pairs.p, pl->d_blkp_beg.p, pl->d_blkp.p, pl->d_fws.p, ada_dev, absd_dev, pl->use_map, pl->m, 1);
      SB_LAUNCH_CHECK_N("ada3_reduce_kernel");
    }
    }
  } else
  for (auto &B : pl->batches) {
    if (B.p1 == B.p0) continue;
    build_tt_kernel<<<B.p1 - B.p0, 256, 0, st>>>(pl->d_pairs.p, B.p0, pl->d_blk_n.p, pl->d_blk_off.p, pl->d_tt_ptr.p, pl->d_tt_col.p,
                                                 pl->d_tt_src.p, pl->d_tt_w.p, pl->d_Atpr.p, udsqr_dev, pl->d_ws.p);
    SB_LAUNCH_CHECK_N("build_tt_kernel");
    if (B.ntiles) {
      gemm_nt_launch(B.ntiles, ctx().sm_count, st, pl->d_descs.p, pl->d_tiles.p + B.tile0, udsqr_dev, pl->d_ws.p, pl->d_ws.p, pl->d_Rlist.p);
      SB_LAUNCH_CHECK_N("gemm_nt_kernel");
    }
    if (B.nsparse) {
      dim3 g((unsigned)std::min((pl->max_nu + 255) / 256, 64), (unsigned)std::min(B.p1 - B.p0, 65535));
      sparse_w_kernel<<<g, 256, 0, st>>>(pl->d_pairs.p, B.p0, B.p1 - B.p0, pl->d_blk_n.p, pl->d_blk_off.p, pl->d_ublk_off.p, pl->d_u_p.p, pl->d_u_q.p,
                                         pl->d_Rlist.p, udsqr_dev, pl->d_ws.p);
      SB_LAUNCH_CHECK_N("sparse_w_kernel");
    }
    {
      static bool attr_done = false;
      if (!attr_done) { SB_CUDA(cudaFuncSetAttribute(ada3_dots_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 225 * 1024)); attr_done = true; }
      ada3_dots_kernel<<<B.p1 - B.p0, 256, pl->dots_smem, st>>>(B.p0, pl->d_adajc.p, pl->d_adair.p, ip, (int)first, pl->d_cpair_beg.p,
          pl->d_pairs.p, pl->d_blk_n.p, pl->d_ublk_off.p, pl->d_blkp_beg.p, pl->d_blkp.p, pl->d_ent_lin.p, pl->d_ent_pk.p,
          pl->d_ent_src.p, pl->d_Atpr.p, pl->herm ? pl->d_ent_scale.p : nullptr, pl->d_ws.p, ada_dev, absd_dev, pl->wcap, pl->use_map, pl->m,
          pl->d_blk_group.p);
    }
    SB_LAUNCH_CHECK_N("ada3_dots_kernel");
    if (B.nmulti) {
      ada3_reduce_kernel<<<B.c1 - B.c0, 256, pl->use_map ? (size_t)pl->m * 4 : 0, st>>>(B.c0, pl->d_adajc.p, pl->d_adair.p, ip, (int)first,
          pl->d_cpair_beg.p, pl->d_pairs.p, pl->d_blkp_beg.p, pl->d_blkp.p, pl->d_ws.p, ada_dev, absd_dev, pl->use_map, pl->m, 0);
      SB_LAUNCH_CHECK_N("ada3_reduce_kernel");
    }
  }
  if (symmetrise) {
    makesym_kernel<<<pl->m, 256, 0, st>>>(pl->m, pl->d_adajc.p, pl->d_adair.p, ada_dev);
    SB_LAUNCH_CHECK_N("makesym_kernel");
  }
  return 0;
}

// ---- host-pointer entries (what the MEX stubs call).  perm: 0-based ordering (Aord.*perm).
int sb200_getada1(sb200_ada_plan *pl, const double *Atpr, const sb_idx *perm, const double *dl, const double *ddet,
                  double *ada_out) {
  static const bool trace = getenv("SB200_TRACE") != nullptr;
  auto now = [] { return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now().time_since_epoch()).count(); };
  double t0 = trace ? now() : 0, t1 = 0, t2 = 0, t3 = 0, t4 = 0;
  SB_TRY(sb200_ada_set_At_values(pl, Atpr));
  if (trace) t1 = now();
  arena_reset();
  const int *ip;
  SB_TRY(set_invperm(pl, perm, &ip));
  double *d_dl = arena<double>((size_t)std::max(pl->lpN, 1)), *d_det = arena<double>((size_t)std::max(pl->nq, 1));
  double *d_out = (double *)mirror_output_slot(sizeof(double) * std::max<long long>(pl->nnzADA, 1));
  SB_CHECK(d_dl && d_det && d_out, "getada1: out of device memory");
  cudaStream_t st = ctx().stream;
  if (pl->lpN) SB_CUDA(cudaMemcpyAsync(d_dl, dl, sizeof(double) * pl->lpN, cudaMemcpyHostToDevice, st));
  if (pl->nq) SB_CUDA(cudaMemcpyAsync(d_det, ddet, sizeof(double) * pl->nq, cudaMemcpyHostToDevice, st));
  if (trace) t2 = now();
  SB_TRY(sb200_getada1_dev(pl, d_dl, d_det, ip, d_out));
  if (trace) { cudaStreamSynchronize(st); t3 = now(); }
  SB_CUDA(cudaMemcpyAsync(ada_out, d_out, sizeof(double) * pl->nnzADA, cudaMemcpyDeviceToHost, st));
  SB_CUDA(cudaStreamSynchronize(st));
  if (trace) t4 = now();
  mirror_publish(d_out, ada_out, sizeof(double) * pl->nnzADA);      // the next plugin call finds ADA on the device
  if (trace) fprintf(stderr, "[getada1] At values %.3f  setup %.3f  kernels %.3f  D2H %.3f  publish %.3f ms\n", t1 - t0, t2 - t1, t3 - t2, t4 - t3, now() - t4);
  return 0;
}

int sb200_getada2(sb200_ada_plan *pl, sb_idx nq, const sb_idx *Qjc, const sb_idx *Qir, const double *Qpr,
                  const sb_idx *perm, const double *ada_in, double *ada_out) {
  arena_reset();
  const int *ip;
  SB_TRY(set_invperm(pl, perm, &ip));
  const int m = pl->m;
  const long long nnzQ = Qjc[m];
  std::vector<long long> jc(Qjc, Qjc + m + 1);
  std::vector<int> ir32;
  SB_TRY(to_i32(Qir, (size_t)nnzQ, ir32, "DAt.q.ir"));
  long long *d_jc = arena<long long>(m + 1);
  int *d_ir = arena<int>((size_t)std::max<long long>(nnzQ, 1));
  double *d_pr = arena<double>((size_t)std::max<long long>(nnzQ, 1));
  double *d_in = (double *)mirror_input(ada_in, sizeof(double) * pl->nnzADA);
  double *d_out = (double *)mirror_output_slot(sizeof(double) * std::max<long long>(pl->nnzADA, 1));
  SB_CHECK(d_jc && d_ir && d_pr && d_in && d_out, "getada2: out of device memory");
  cudaStream_t st = ctx().stream;
  SB_CUDA(cudaMemcpyAsync(d_jc, jc.data(), sizeof(long long) * (m + 1), cudaMemcpyHostToDevice, st));
  if (nnzQ) {
    SB_CUDA(cudaMemcpyAsync(d_ir, ir32.data(), sizeof(int) * nnzQ, cudaMemcpyHostToDevice, st));
    SB_CUDA(cudaMemcpyAsync(d_pr, Qpr, sizeof(double) * nnzQ, cudaMemcpyHostToDevice, st));
  }
  SB_TRY(getada2_impl(pl, d_jc, d_ir, d_pr, nnzQ, ip, d_in, d_out));
  SB_CUDA(cudaMemcpyAsync(ada_out, d_out, sizeof(double) * pl->nnzADA, cudaMemcpyDeviceToHost, st));
  SB_CUDA(cudaStreamSynchronize(st));
  mirror_publish(d_out, ada_out, sizeof(double) * pl->nnzADA);
  (void)nq;
  return 0;
}

int sb200_getada3(sb200_ada_plan *pl, const double *Atpr, const double *udsqr, sb_idx lenud, const sb_idx *perm,
                  sb_idx first, const double *ada_in, double *ada_out, double *absd_out) {
  SB_TRY(sb200_ada_set_At_values(pl, Atpr));
  arena_reset();
  const int *ip;
  SB_TRY(set_invperm(pl, perm, &ip));
  double *d_ud = arena<double>((size_t)std::max<long long>(lenud, 1));
  const double *d_in = (const double *)mirror_input(ada_in, sizeof(double) * pl->nnzADA);
  double *d_ada = (double *)mirror_output_slot(sizeof(double) * std::max<long long>(pl->nnzADA, 1));
  double *d_absd = arena<double>((size_t)std::max(pl->m, 1));
  SB_CHECK(d_ud && d_in && d_ada && d_absd, "getada3: out of device memory");
  cudaStream_t st = ctx().stream;
  if (lenud) SB_CUDA(cudaMemcpyAsync(d_ud, udsqr, sizeof(double) * lenud, cudaMemcpyHostToDevice, st));
  SB_CUDA(cudaMemcpyAsync(d_ada, d_in, sizeof(double) * pl->nnzADA, cudaMemcpyDeviceToDevice, st));
  SB_TRY(sb200_getada3_dev(pl, d_ud, ip, first, d_ada, d_absd, 1));
  SB_CUDA(cudaMemcpyAsync(ada_out, d_ada, sizeof(double) * pl->nnzADA, cudaMemcpyDeviceToHost, st));
  SB_CUDA(cudaMemcpyAsync(absd_out, d_absd, sizeof(double) * pl->m, cudaMemcpyDeviceToHost, st));
  SB_CUDA(cudaStreamSynchronize(st));
  mirror_publish(d_ada, ada_out, sizeof(double) * pl->nnzADA);
  return 0;
}

}  // extern "C"
