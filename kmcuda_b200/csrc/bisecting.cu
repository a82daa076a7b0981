// bisecting.cu -- device side of bisecting k-means (scikit-learn's BisectingKMeans; Job::bisecting in job.cu, DESIGN.md
// §4o).  The nodes of the tree are ranges [lo, hi) of a permutation `perm` of the rows, each holding its rows in
// ascending order.  One wave bisects many leaves at once: every (node, init r) pair is a segment, and the CTAs of a
// launch map onto (segment, chunk) pairs through a table the host builds (uint2 {segment, chunk}).  A chunk is kBkChunk
// consecutive positions of a segment's range; every double total is a sequential sum in position order inside a chunk,
// then the chunks in order, so nothing depends on the launch shape or on which other segments share the wave.
//   keys     random init: the two positive-weight rows of smallest -ln(u) / w per chunk, folded per segment; greedy
//            init: c0 = the smallest, then distances, trial keys, trial potentials and the pick (§4m's round 1)
//   step     one pass over the rows: the reference argmin between the two centres, e = the Kahan sum of (x - c)^2 to
//            the winner, the label byte, and per chunk and child S = sum w x, W = sum w, I = sum w e, plus the row
//            counts, changed labels and the farthest positive-weight row
//   fold     per segment: the chunks in order, scikit-learn's relocation of an empty child, the new centres, their
//            squared norms and sum ||dc||^2, into one status record per segment
//   split    flags of child 0, one exclusive scan over perm, one stable scatter of every split node of a round
//   assign   assign[perm[p]] = the index of the leaf holding position p
#include <cub/device/device_scan.cuh>

#include <cmath>

#include "exact.cuh"
#include "fixed_order.cuh"
#include "kernels.h"

namespace kmb {

namespace {

constexpr int kBkRows = kStagedRows;   // threads per CTA of the row kernels, rows per staged sub-tile
constexpr int kBkFoldThreads = 256;

struct KeyPair {
  double k;
  uint32_t row;
};

__device__ __forceinline__ bool key_less(double ka, uint32_t ra, double kb, uint32_t rb) {
  return ka < kb || (ka == kb && ra < rb);
}

__device__ __forceinline__ void top2_push(KeyPair& a, KeyPair& b, double k, uint32_t row) {
  if (key_less(k, row, a.k, a.row)) {
    b = a;
    a = {k, row};
  } else if (key_less(k, row, b.k, b.row)) {
    b = {k, row};
  }
}

// the draw key of stage `stage` of init r of node [lo, hi) (bk_node_key)
__host__ __device__ __forceinline__ uint64_t bk_key(uint32_t seed, uint32_t lo, uint32_t hi, uint32_t r,
                                                    uint32_t stage) {
  uint64_t k = splitmix64(kBkTagNode ^ seed);
  k = splitmix64(k + lo);
  k = splitmix64(k + hi);
  return splitmix64(k + ((static_cast<uint64_t>(r) << 8) | stage));
}

// one feature of the step kernel's four chains: the dots with both centres and the squared differences to both
__device__ __forceinline__ void step_chains(Kahan& d0, Kahan& d1, Kahan& e0, Kahan& e1, float x, float a, float b) {
  d0.mac(x, a);
  d1.mac(x, b);
  e0.sqdiff(x, a);
  e1.sqdiff(x, b);
}

__device__ __forceinline__ const float* seg_centres(const float* cbuf, uint32_t slot, int D) {
  return cbuf + static_cast<size_t>(slot) * 2 * D;
}

// -ln(u) / w of every positive-weight row of the chunk; the chunk's two smallest (key, row) go to ckeys[2 * chunk]
__global__ void __launch_bounds__(kBkRows)
bk_keys_kernel(const float* __restrict__ w, const uint32_t* __restrict__ perm, const BkSeg* __restrict__ segs,
               const uint2* __restrict__ work, BkKey* __restrict__ ckeys) {
  __shared__ KeyPair s_k[2 * kBkRows];
  const uint2 wk = work[blockIdx.x];
  const BkSeg sg = segs[wk.x];
  const uint32_t c0 = sg.lo + wk.y * kBkChunk, c1 = min(sg.hi, c0 + kBkChunk);
  KeyPair a = {INFINITY, UINT32_MAX}, b = {INFINITY, UINT32_MAX};
  for (uint32_t p = c0 + threadIdx.x; p < c1; p += kBkRows) {
    const uint32_t row = perm[p];
    const float wi = w ? w[row] : 1.f;
    if (wi > 0.f) top2_push(a, b, -log(unit_oo(splitmix64(sg.key ^ row))) / static_cast<double>(wi), row);
  }
  s_k[2 * threadIdx.x] = a;
  s_k[2 * threadIdx.x + 1] = b;
  __syncthreads();
  if (threadIdx.x == 0) {
    KeyPair x = {INFINITY, UINT32_MAX}, y = {INFINITY, UINT32_MAX};
    for (int q = 0; q < 2 * kBkRows; q++) top2_push(x, y, s_k[q].k, s_k[q].row);
    BkKey* out = ckeys + 2 * (static_cast<size_t>(sg.pbase) + wk.y);
    out[0] = {x.k, x.row, 0u};
    out[1] = {y.k, y.row, 0u};
  }
}

// the init keys of every segment folded over its chunks: random init, centres 0 / 1 = the rows of the two smallest keys;
// greedy (`greedy`), centre 0 = the row of the smallest key (c0), centre 1 comes from bk_gpick_kernel.  status->init_row
// = the two rows (init_row[1] = UINT32_MAX: no init, the node cannot be split)
__global__ void __launch_bounds__(kBkFoldThreads)
bk_init_fold_kernel(const float* __restrict__ X, int D, const BkSeg* __restrict__ segs, const BkKey* __restrict__ ckeys,
                    bool greedy, float* __restrict__ cbuf, float* __restrict__ csqbuf, BkStatus* __restrict__ status) {
  __shared__ uint32_t s_rows[2];
  const BkSeg sg = segs[blockIdx.x];
  const uint32_t nch = (sg.hi - sg.lo + kBkChunk - 1) / kBkChunk;
  if (threadIdx.x == 0) {
    KeyPair x = {INFINITY, UINT32_MAX}, y = {INFINITY, UINT32_MAX};
    for (uint32_t q = 0; q < 2 * nch; q++) {
      const BkKey k = ckeys[2 * static_cast<size_t>(sg.pbase) + q];
      top2_push(x, y, k.key, k.row);
    }
    s_rows[0] = x.row;
    s_rows[1] = y.row;
  }
  __syncthreads();
  const uint32_t r0 = s_rows[0], r1 = s_rows[1];
  BkStatus* st = status + blockIdx.x;
  if (threadIdx.x == 0) {
    *st = BkStatus{};
    st->init_row[0] = r0;
    st->init_row[1] = greedy ? (r0 == UINT32_MAX ? UINT32_MAX : 0u) : r1;
  }
  // random: fewer than two positive-weight rows, greedy: none; the node cannot be split
  if (greedy ? r0 == UINT32_MAX : r1 == UINT32_MAX) return;
  float* C = cbuf + static_cast<size_t>(sg.cur) * 2 * D;
  for (int f = threadIdx.x; f < D; f += kBkFoldThreads) {
    C[f] = X[static_cast<size_t>(r0) * D + f];
    if (!greedy) C[D + f] = X[static_cast<size_t>(r1) * D + f];
  }
  __syncthreads();
  if (threadIdx.x == 0) csqbuf[2 * sg.cur] = csqr_exact<0>(C, D);
  if (threadIdx.x == 32 && !greedy) csqbuf[2 * sg.cur + 1] = csqr_exact<0>(C + D, D);
}

// ---- greedy k-means++ init (§4m's round 1 restricted to the node): c0 from bk_keys_kernel / bk_init_fold_kernel, then
// d = the true distance to c0, mass m = w d^2, trial t = the row of smallest -ln(u_t) / m (stage 1 + t), phi_t = the
// fixed-order sum of mass(min(d, e_t)), the lowest phi_t (then t) is centre 1.

__device__ __forceinline__ bool seg_live(const BkStatus* status, uint32_t s) { return status[s].init_row[1] != UINT32_MAX; }

// the minimum (key, row) over the CTA's threads into *best (thread 0, combined with what *best holds)
__device__ __forceinline__ void cta_min(double k, uint32_t row, KeyPair* s_warp, KeyPair* best) {
  for (int o = 16; o > 0; o >>= 1) {
    const double ok = __shfl_down_sync(0xffffffffu, k, o);
    const uint32_t orow = __shfl_down_sync(0xffffffffu, row, o);
    if (key_less(ok, orow, k, row)) {
      k = ok;
      row = orow;
    }
  }
  if ((threadIdx.x & 31) == 0) s_warp[threadIdx.x >> 5] = {k, row};
  __syncthreads();
  if (threadIdx.x == 0)
    for (int q = 0; q < kBkRows / 32; q++)
      if (key_less(s_warp[q].k, s_warp[q].row, best->k, best->row)) *best = s_warp[q];
  __syncthreads();
}

// d of every row (dist[r][position]) and the chunk's smallest trial key per trial into tkeys[chunk][t]
template <bool VEC4>
__global__ void __launch_bounds__(kBkRows)
bk_gdist_kernel(const float* __restrict__ X, int D, const float* __restrict__ w, const uint32_t* __restrict__ perm,
                uint32_t N, const BkSeg* __restrict__ segs, const uint2* __restrict__ work,
                const float* __restrict__ cbuf, const BkStatus* __restrict__ status, uint32_t L,
                float* __restrict__ dist, BkKey* __restrict__ tkeys) {
  __shared__ uint32_t s_row[kBkRows];
  __shared__ float tile[kBkRows * 33];
  __shared__ KeyPair s_warp[kBkRows / 32], s_best[kGppMaxTrials];
  const int t = threadIdx.x;
  const uint2 wk = work[blockIdx.x];
  if (!seg_live(status, wk.x)) return;
  const BkSeg sg = segs[wk.x];
  const uint32_t c0 = sg.lo + wk.y * kBkChunk, c1 = min(sg.hi, c0 + kBkChunk);
  const float* C0 = seg_centres(cbuf, sg.cur, D);
  if (t < static_cast<int>(L)) s_best[t] = {INFINITY, UINT32_MAX};
  for (uint32_t p0 = c0; p0 < c1; p0 += kBkRows) {
    const uint32_t n = min(c1 - p0, static_cast<uint32_t>(kBkRows));
    const bool live = static_cast<uint32_t>(t) < n;
    s_row[t] = live ? perm[p0 + t] : 0u;
    __syncthreads();
    const float d = finalize_distance<0>(staged_own_sum<VEC4, 0>(X, s_row, 0u, n, D, C0, live, tile));
    const uint32_t row = s_row[t];
    double m = 0.0;
    if (live) {
      dist[static_cast<size_t>(sg.r) * N + p0 + t] = d;
      m = d2_mass(d, w ? w[row] : 1.f);
    }
    for (uint32_t q = 0; q < L; q++) {
      const uint64_t key = bk_key(sg.seed, sg.lo, sg.hi, sg.r, 1 + q);
      const double k = m > 0.0 ? -log(unit_oo(splitmix64(key ^ row))) / m : INFINITY;
      cta_min(k, m > 0.0 ? row : UINT32_MAX, s_warp, s_best + q);
    }
  }
  if (t < static_cast<int>(L)) {
    const KeyPair b = s_best[t];
    tkeys[(static_cast<size_t>(sg.pbase) + wk.y) * kGppMaxTrials + t] = {b.k, b.row, 0u};
  }
}

// one CTA per segment: trows[seg][t] = the trial rows (UINT32_MAX for every t when no row has mass: no init)
__global__ void bk_gfold_kernel(const BkSeg* __restrict__ segs, const BkKey* __restrict__ tkeys, uint32_t L,
                                BkStatus* __restrict__ status, uint32_t* __restrict__ trows) {
  const uint32_t t = threadIdx.x;
  if (!seg_live(status, blockIdx.x) || t >= L) return;
  const BkSeg sg = segs[blockIdx.x];
  const uint32_t nch = (sg.hi - sg.lo + kBkChunk - 1) / kBkChunk;
  KeyPair b = {INFINITY, UINT32_MAX};
  for (uint32_t q = 0; q < nch; q++) {
    const BkKey k = tkeys[(static_cast<size_t>(sg.pbase) + q) * kGppMaxTrials + t];
    if (key_less(k.key, k.row, b.k, b.row)) b = {k.key, k.row};
  }
  trows[static_cast<size_t>(blockIdx.x) * kGppMaxTrials + t] = b.row;
  if (t == 0 && b.row == UINT32_MAX) status[blockIdx.x].init_row[1] = UINT32_MAX;   // no mass left
}

// the chunk's sum of mass(min(d, e_t)) per trial, in position order, into phi[chunk][t]
template <bool VEC4>
__global__ void __launch_bounds__(kBkRows)
bk_gtrial_kernel(const float* __restrict__ X, int D, const float* __restrict__ w, const uint32_t* __restrict__ perm,
                 uint32_t N, const BkSeg* __restrict__ segs, const uint2* __restrict__ work,
                 const BkStatus* __restrict__ status, const uint32_t* __restrict__ trows, uint32_t L,
                 const float* __restrict__ dist, double* __restrict__ phi) {
  __shared__ uint32_t s_row[kBkRows];
  __shared__ float tile[kBkRows * 33];
  __shared__ double s_m[kBkRows], s_phi[kGppMaxTrials];
  const int t = threadIdx.x;
  const uint2 wk = work[blockIdx.x];
  if (!seg_live(status, wk.x)) return;
  const BkSeg sg = segs[wk.x];
  const uint32_t c0 = sg.lo + wk.y * kBkChunk, c1 = min(sg.hi, c0 + kBkChunk);
  if (t < static_cast<int>(L)) s_phi[t] = 0.0;
  for (uint32_t p0 = c0; p0 < c1; p0 += kBkRows) {
    const uint32_t n = min(c1 - p0, static_cast<uint32_t>(kBkRows));
    const bool live = static_cast<uint32_t>(t) < n;
    s_row[t] = live ? perm[p0 + t] : 0u;
    const float d = live ? dist[static_cast<size_t>(sg.r) * N + p0 + t] : 0.f;
    const float wi = live ? (w ? w[s_row[t]] : 1.f) : 0.f;
    __syncthreads();
    for (uint32_t q = 0; q < L; q++) {
      const float* T = X + static_cast<size_t>(trows[static_cast<size_t>(wk.x) * kGppMaxTrials + q]) * D;
      const float e = finalize_distance<0>(staged_own_sum<VEC4, 0>(X, s_row, 0u, n, D, T, live, tile));
      s_m[t] = live ? d2_mass(e < d ? e : d, wi) : 0.0;
      __syncthreads();
      if (t == 0) {
        double a = s_phi[q];
        for (uint32_t r = 0; r < n; r++) a = __dadd_rn(a, s_m[r]);
        s_phi[q] = a;
      }
      __syncthreads();
    }
  }
  if (t < static_cast<int>(L)) phi[(static_cast<size_t>(sg.pbase) + wk.y) * kGppMaxTrials + t] = s_phi[t];
}

// one CTA per segment: phi_t folded over the chunks in order, the lowest (then the lowest t) gives centre 1
__global__ void __launch_bounds__(kBkFoldThreads)
bk_gpick_kernel(const float* __restrict__ X, int D, const BkSeg* __restrict__ segs, const uint32_t* __restrict__ trows,
                uint32_t L, const double* __restrict__ phi, float* __restrict__ cbuf, float* __restrict__ csqbuf,
                BkStatus* __restrict__ status) {
  __shared__ uint32_t s_pick;
  if (!seg_live(status, blockIdx.x)) return;
  const BkSeg sg = segs[blockIdx.x];
  const uint32_t nch = (sg.hi - sg.lo + kBkChunk - 1) / kBkChunk;
  if (threadIdx.x == 0) {
    uint32_t best = 0;
    double bphi = 0.0;
    for (uint32_t q = 0; q < L; q++) {
      double a = 0.0;
      for (uint32_t c = 0; c < nch; c++) a = __dadd_rn(a, phi[(static_cast<size_t>(sg.pbase) + c) * kGppMaxTrials + q]);
      if (q == 0 || a < bphi) {
        best = q;
        bphi = a;
      }
    }
    s_pick = trows[static_cast<size_t>(blockIdx.x) * kGppMaxTrials + best];
    status[blockIdx.x].init_row[1] = s_pick;
  }
  __syncthreads();
  const uint32_t r1 = s_pick;
  float* C = cbuf + static_cast<size_t>(sg.cur) * 2 * D;
  for (int f = threadIdx.x; f < D; f += kBkFoldThreads) C[D + f] = X[static_cast<size_t>(r1) * D + f];
  __syncthreads();
  if (threadIdx.x == 0) csqbuf[2 * sg.cur + 1] = csqr_exact<0>(C + D, D);
}

// One E step over a chunk of a segment, kBkRows rows at a time (staged as staged_own_sum stages them), and the chunk's
// sums of the M step.  The columns of a chunk's partial are, per child j, [S_0 .. S_{D-1}, W, I] at j * (D + 2), then
// the chunk's sum of w e over all rows at 2 (D + 2).  The member sums re-read the sub-tile's rows, which the staged
// pass has just brought into L2.  mode kBkFinal (E step only) skips the S columns.
template <bool VEC4>
__global__ void __launch_bounds__(kBkRows, 8)
bk_step_kernel(const float* __restrict__ X, int D, const float* __restrict__ w, const uint32_t* __restrict__ perm,
               uint8_t* __restrict__ lab, uint32_t N, const BkSeg* __restrict__ segs, const uint2* __restrict__ work,
               const float* __restrict__ cbuf, const float* __restrict__ csqbuf, double* __restrict__ part,
               BkChunkStat* __restrict__ cstat) {
  __shared__ uint32_t s_row[kBkRows];
  __shared__ float tile[kBkRows * 33];
  __shared__ double s_w[kBkRows], s_we[kBkRows];
  __shared__ uint8_t s_lab[kBkRows];
  __shared__ uint32_t s_cnt[2], s_npos[2], s_changed;
  __shared__ unsigned long long s_fk[2];
  const int t = threadIdx.x;
  const uint2 wk = work[blockIdx.x];
  const BkSeg sg = segs[wk.x];
  const uint32_t c0 = sg.lo + wk.y * kBkChunk, c1 = min(sg.hi, c0 + kBkChunk);
  const float* C0 = seg_centres(cbuf, sg.cur, D);
  const float* C1 = C0 + D;
  const float q0 = csqbuf[2 * sg.cur], q1 = csqbuf[2 * sg.cur + 1];
  uint8_t* L = lab + static_cast<size_t>(sg.r) * N;
  const int ncol = D + 2;
  double* P = part + static_cast<size_t>(sg.pbase + wk.y) * (2 * ncol + 1);
  if (t < 2) {
    s_cnt[t] = 0;
    s_npos[t] = 0;
    s_fk[t] = 0;
  }
  if (t == 0) s_changed = 0;
  const int first_col = sg.mode == kBkFinal ? D : 0;
  for (uint32_t p0 = c0; p0 < c1; p0 += kBkRows) {
    const uint32_t n = min(c1 - p0, static_cast<uint32_t>(kBkRows));
    const bool live = static_cast<uint32_t>(t) < n;
    s_row[t] = live ? perm[p0 + t] : 0u;
    __syncthreads();
    Kahan d0, d1, e0, e1;
    for (int f0 = 0; f0 < D; f0 += 32) {
      const int fl = min(32, D - f0);
      stage_slice(X, s_row, 0u, n, D, f0, fl, tile);
      __syncthreads();
      if (live) {
        const float* xs = tile + t * 33;
        if (VEC4 && fl == 32) {   // the centres as float4 (D % 4 == 0), the same order of operations
#pragma unroll
          for (int q = 0; q < 8; q++) {
            const float4 a = __ldg(reinterpret_cast<const float4*>(C0 + f0) + q);
            const float4 b = __ldg(reinterpret_cast<const float4*>(C1 + f0) + q);
            step_chains(d0, d1, e0, e1, xs[4 * q], a.x, b.x);
            step_chains(d0, d1, e0, e1, xs[4 * q + 1], a.y, b.y);
            step_chains(d0, d1, e0, e1, xs[4 * q + 2], a.z, b.z);
            step_chains(d0, d1, e0, e1, xs[4 * q + 3], a.w, b.w);
          }
        } else {
          for (int f = 0; f < fl; f++) step_chains(d0, d1, e0, e1, xs[f], __ldg(C0 + f0 + f), __ldg(C1 + f0 + f));
        }
      }
      __syncthreads();
    }
    if (live) {
      const uint32_t row = s_row[t];
      // the reference argmin of two centres: strict <, ties to centre 0
      const uint8_t lb = lloyd_score<0>(d1.sum, q1) < lloyd_score<0>(d0.sum, q0) ? 1 : 0;
      const float e = lb ? e1.sum : e0.sum;
      const float wi = w ? w[row] : 1.f;
      if (L[p0 + t] != lb) atomicAdd(&s_changed, 1u);
      L[p0 + t] = lb;
      atomicAdd(&s_cnt[lb], 1u);
      if (wi > 0.f) {
        atomicAdd(&s_npos[lb], 1u);
        atomicMax(&s_fk[lb], (static_cast<unsigned long long>(__float_as_uint(e)) << 32) | (~row & 0xFFFFFFFFu));
      }
      s_lab[t] = lb;
      s_w[t] = static_cast<double>(wi);
      s_we[t] = __dmul_rn(static_cast<double>(wi), static_cast<double>(e));
    }
    __syncthreads();
    const bool fresh = p0 == c0;
    for (int c = first_col + t; c < D + 3; c += kBkRows) {
      if (c == D + 2) {
        double a = fresh ? 0.0 : P[2 * ncol];
        for (uint32_t r = 0; r < n; r++) a = __dadd_rn(a, s_we[r]);
        P[2 * ncol] = a;
        continue;
      }
      double a0 = fresh ? 0.0 : P[c], a1 = fresh ? 0.0 : P[ncol + c];
      if (c < D) {
        for (uint32_t r = 0; r < n; r++) {
          const double v = __dmul_rn(s_w[r], static_cast<double>(X[static_cast<size_t>(s_row[r]) * D + c]));
          if (s_lab[r]) a1 = __dadd_rn(a1, v);
          else a0 = __dadd_rn(a0, v);
        }
      } else {
        const double* src = c == D ? s_w : s_we;
        for (uint32_t r = 0; r < n; r++) {
          if (s_lab[r]) a1 = __dadd_rn(a1, src[r]);
          else a0 = __dadd_rn(a0, src[r]);
        }
      }
      P[c] = a0;
      P[ncol + c] = a1;
    }
    __syncthreads();
  }
  if (t == 0) {
    BkChunkStat s;
    s.fk[0] = s_fk[0];
    s.fk[1] = s_fk[1];
    s.cnt[0] = s_cnt[0];
    s.cnt[1] = s_cnt[1];
    s.npos[0] = s_npos[0];
    s.npos[1] = s_npos[1];
    s.changed = s_changed;
    s.pad = 0;
    cstat[sg.pbase + wk.y] = s;
  }
}

// the fixed-order fold of column `col` over a segment's chunks
__device__ __forceinline__ double fold_col(const double* __restrict__ P, size_t stride, uint32_t nch, int col) {
  double a = 0.0;
  for (uint32_t q = 0; q < nch; q++) a = __dadd_rn(a, P[q * stride + col]);
  return a;
}

// One CTA per segment: fold the chunks, apply the empty-child rule, write the new centres into slot sg.nxt with their
// squared norms, and the status record
__global__ void __launch_bounds__(kBkFoldThreads)
bk_fold_kernel(const float* __restrict__ X, int D, const float* __restrict__ w, const BkSeg* __restrict__ segs,
               const double* __restrict__ part, const BkChunkStat* __restrict__ cstat, float* __restrict__ cbuf,
               float* __restrict__ csqbuf, BkStatus* __restrict__ status) {
  __shared__ double s_tot[5];   // W0, W1, I0, I1, I
  __shared__ double s_W[2], s_rw;
  __shared__ uint32_t s_rrow, s_rj;
  const int t = threadIdx.x;
  const BkSeg sg = segs[blockIdx.x];
  const uint32_t nch = (sg.hi - sg.lo + kBkChunk - 1) / kBkChunk;
  const int ncol = D + 2;
  const size_t stride = 2 * static_cast<size_t>(ncol) + 1;
  const double* P = part + static_cast<size_t>(sg.pbase) * stride;
  BkStatus* st = status + blockIdx.x;
  if (t < 5) {
    const int col = t == 4 ? 2 * ncol : (t & 1) * ncol + D + (t >> 1);
    s_tot[t] = fold_col(P, stride, nch, col);
  }
  __syncthreads();
  if (t == 0) {
    BkStatus s = BkStatus{};
    unsigned long long fk[2] = {0, 0};
    for (uint32_t q = 0; q < nch; q++) {
      const BkChunkStat c = cstat[sg.pbase + q];
      for (int j = 0; j < 2; j++) {
        s.cnt[j] += c.cnt[j];
        s.npos[j] += c.npos[j];
        fk[j] = max(fk[j], c.fk[j]);
      }
      s.changed += c.changed;
    }
    s.W[0] = s_tot[0];
    s.W[1] = s_tot[1];
    s.I[0] = s_tot[2];
    s.I[1] = s_tot[3];
    s.inertia = s_tot[4];
    // scikit-learn's _relocate_empty_clusters_dense for k = 2: the empty child takes the donor's farthest row
    s_rj = UINT32_MAX;
    s_W[0] = s.W[0];
    s_W[1] = s.W[1];
    if (sg.mode != kBkFinal) {
      for (int j = 0; j < 2; j++) {
        if (s.W[j] == 0.0 && s.npos[1 - j] >= 2) {
          const uint32_t row = ~static_cast<uint32_t>(fk[1 - j] & 0xFFFFFFFFu);
          s_rj = j;
          s_rrow = row;
          s_rw = static_cast<double>(w ? w[row] : 1.f);
          s_W[1 - j] = __dsub_rn(s_W[1 - j], s_rw);
          s_W[j] = s_rw;
          s.relocated = 1;
          s.init_row[0] = row;
          break;
        }
      }
    }
    *st = s;
  }
  __syncthreads();
  if (sg.mode == kBkFinal) return;
  const float* Co = seg_centres(cbuf, sg.cur, D);
  float* Cn = cbuf + static_cast<size_t>(sg.nxt) * 2 * D;
  const uint32_t rj = s_rj;
  for (int f = t; f < D; f += kBkFoldThreads) {
    double S[2] = {fold_col(P, stride, nch, f), fold_col(P, stride, nch, ncol + f)};
    if (rj != UINT32_MAX) {
      const double v = __dmul_rn(s_rw, static_cast<double>(X[static_cast<size_t>(s_rrow) * D + f]));
      S[1 - rj] = __dsub_rn(S[1 - rj], v);
      S[rj] = v;
    }
    for (int j = 0; j < 2; j++)   // a child left without weight keeps its centre
      Cn[j * D + f] = s_W[j] > 0.0 ? static_cast<float>(__ddiv_rn(S[j], s_W[j])) : Co[j * D + f];
  }
  __syncthreads();
  if (t == 0) csqbuf[2 * sg.nxt] = csqr_exact<0>(Cn, D);
  if (t == 32) csqbuf[2 * sg.nxt + 1] = csqr_exact<0>(Cn + D, D);
  if (t == 64) {   // sum ||c_new - c_old||^2 in double: child 0's features in order, then child 1's
    double a = 0.0;
    for (int f = 0; f < 2 * D; f++) {
      const double d = __dsub_rn(static_cast<double>(Cn[f]), static_cast<double>(Co[f]));
      a = __dadd_rn(a, __dmul_rn(d, d));
    }
    st->shift = a;
  }
}

// flags[p] = 1 for the child-0 positions of the split nodes (segments) of a round
__global__ void __launch_bounds__(kBkRows)
bk_flag_kernel(const uint8_t* __restrict__ lab, uint32_t N, const BkSeg* __restrict__ segs,
               const uint2* __restrict__ work, uint32_t* __restrict__ flags) {
  const uint2 wk = work[blockIdx.x];
  const BkSeg sg = segs[wk.x];
  const uint32_t c0 = sg.lo + wk.y * kBkChunk, c1 = min(sg.hi, c0 + kBkChunk);
  const uint8_t* L = lab + static_cast<size_t>(sg.r) * N;
  for (uint32_t p = c0 + threadIdx.x; p < c1; p += kBkRows) flags[p] = L[p] == 0;
}

// stable partition of every split node: child 0's rows first, then child 1's, each in position order
__global__ void __launch_bounds__(kBkRows)
bk_scatter_kernel(const uint32_t* __restrict__ perm, const uint32_t* __restrict__ flags,
                  const uint32_t* __restrict__ excl, const BkSeg* __restrict__ segs, const uint2* __restrict__ work,
                  uint32_t* __restrict__ out) {
  const uint2 wk = work[blockIdx.x];
  const BkSeg sg = segs[wk.x];
  const uint32_t c0 = sg.lo + wk.y * kBkChunk, c1 = min(sg.hi, c0 + kBkChunk);
  const uint32_t base = excl[sg.lo], n0 = excl[sg.hi] - base;
  for (uint32_t p = c0 + threadIdx.x; p < c1; p += kBkRows) {
    const uint32_t k = excl[p] - base;
    out[flags[p] ? sg.lo + k : sg.lo + n0 + (p - sg.lo - k)] = perm[p];
  }
}

// assign[perm[p]] = the leaf whose range holds p (leaf_lo ascending, leaf_lo[0] = 0)
__global__ void bk_assign_kernel(const uint32_t* __restrict__ perm, uint32_t N, const uint32_t* __restrict__ leaf_lo,
                                 uint32_t K, uint32_t* __restrict__ assign) {
  const uint32_t p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= N) return;
  uint32_t lo = 0, hi = K;   // the last leaf with leaf_lo <= p
  while (hi - lo > 1) {
    const uint32_t mid = (lo + hi) / 2;
    if (leaf_lo[mid] <= p) lo = mid;
    else hi = mid;
  }
  assign[perm[p]] = lo;
}

__global__ void bk_iota_kernel(uint32_t* __restrict__ p, uint32_t n) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) p[i] = i;
}

}  // namespace

uint64_t bk_node_key(uint32_t seed, uint32_t lo, uint32_t hi, uint32_t r, uint32_t stage) {
  return bk_key(seed, lo, hi, r, stage);
}

size_t bk_partial_doubles(int D) { return 2 * (static_cast<size_t>(D) + 2) + 1; }

cudaError_t launch_bk_iota(uint32_t* perm, uint32_t n, cudaStream_t st) {
  bk_iota_kernel<<<cdiv(n, 256), 256, 0, st>>>(perm, n);
  return cudaGetLastError();
}

cudaError_t launch_bk_init(const BkLaunch& a, uint32_t L, cudaStream_t st) {
  const bool greedy = L > 0;
  bk_keys_kernel<<<a.nwork, kBkRows, 0, st>>>(a.w, a.perm, a.segs, a.work, a.keys);
  bk_init_fold_kernel<<<a.nseg, kBkFoldThreads, 0, st>>>(a.X, a.D, a.segs, a.keys, greedy, a.cbuf, a.csq, a.status);
  if (!greedy) return cudaGetLastError();
  if (a.D % 4 == 0)
    bk_gdist_kernel<true><<<a.nwork, kBkRows, 0, st>>>(a.X, a.D, a.w, a.perm, a.N, a.segs, a.work, a.cbuf, a.status,
                                                       L, a.dist, a.tkeys);
  else
    bk_gdist_kernel<false><<<a.nwork, kBkRows, 0, st>>>(a.X, a.D, a.w, a.perm, a.N, a.segs, a.work, a.cbuf, a.status,
                                                        L, a.dist, a.tkeys);
  bk_gfold_kernel<<<a.nseg, 32, 0, st>>>(a.segs, a.tkeys, L, a.status, a.trows);
  if (a.D % 4 == 0)
    bk_gtrial_kernel<true><<<a.nwork, kBkRows, 0, st>>>(a.X, a.D, a.w, a.perm, a.N, a.segs, a.work, a.status, a.trows,
                                                        L, a.dist, a.phi);
  else
    bk_gtrial_kernel<false><<<a.nwork, kBkRows, 0, st>>>(a.X, a.D, a.w, a.perm, a.N, a.segs, a.work, a.status,
                                                         a.trows, L, a.dist, a.phi);
  bk_gpick_kernel<<<a.nseg, kBkFoldThreads, 0, st>>>(a.X, a.D, a.segs, a.trows, L, a.phi, a.cbuf, a.csq, a.status);
  return cudaGetLastError();
}

cudaError_t launch_bk_step(const BkLaunch& a, cudaStream_t st) {
  if (a.D % 4 == 0)
    bk_step_kernel<true><<<a.nwork, kBkRows, 0, st>>>(a.X, a.D, a.w, a.perm, a.lab, a.N, a.segs, a.work, a.cbuf,
                                                      a.csq, a.part, a.cstat);
  else
    bk_step_kernel<false><<<a.nwork, kBkRows, 0, st>>>(a.X, a.D, a.w, a.perm, a.lab, a.N, a.segs, a.work, a.cbuf,
                                                       a.csq, a.part, a.cstat);
  bk_fold_kernel<<<a.nseg, kBkFoldThreads, 0, st>>>(a.X, a.D, a.w, a.segs, a.part, a.cstat, a.cbuf, a.csq, a.status);
  return cudaGetLastError();
}

size_t bk_split_bytes(uint32_t N) {
  size_t b = 0;
  cub::DeviceScan::ExclusiveSum(nullptr, b, static_cast<const uint32_t*>(nullptr), static_cast<uint32_t*>(nullptr),
                                N + 1);
  return b;
}

cudaError_t launch_bk_split(const BkLaunch& a, uint32_t* flags, uint32_t* excl, void* tmp, size_t tmp_bytes,
                            uint32_t* perm_out, cudaStream_t st) {
  cudaError_t e;
  if ((e = cudaMemsetAsync(flags, 0, sizeof(uint32_t) * (a.N + 1), st)) != cudaSuccess) return e;
  if ((e = cudaMemcpyAsync(perm_out, a.perm, sizeof(uint32_t) * a.N, cudaMemcpyDeviceToDevice, st)) != cudaSuccess)
    return e;
  bk_flag_kernel<<<a.nwork, kBkRows, 0, st>>>(a.lab, a.N, a.segs, a.work, flags);
  if ((e = cudaGetLastError()) != cudaSuccess) return e;
  size_t bytes = tmp_bytes;
  if ((e = cub::DeviceScan::ExclusiveSum(tmp, bytes, flags, excl, a.N + 1, st)) != cudaSuccess) return e;
  bk_scatter_kernel<<<a.nwork, kBkRows, 0, st>>>(a.perm, flags, excl, a.segs, a.work, perm_out);
  return cudaGetLastError();
}

cudaError_t launch_bk_assign(const uint32_t* perm, uint32_t N, const uint32_t* leaf_lo, uint32_t K, uint32_t* assign,
                             cudaStream_t st) {
  bk_assign_kernel<<<cdiv(N, 256), 256, 0, st>>>(perm, N, leaf_lo, K, assign);
  return cudaGetLastError();
}

}  // namespace kmb
