// greedy_plusplus.cu -- device side of the greedy k-means++ seeding (scikit-learn's _kmeans_plusplus: d^2 draws, several
// local trials per round, the trial that lowers the potential most wins; DESIGN.md §4m).
//
// A round of the seeding (Job::init_greedy_plusplus, seeding.cu) is
//   draw      fold the previous round's winner into d (d = d'_winner, d = 0 on the chosen row), m_i = w_i d_i^2, and the
//             per-block (key, row) minima of the round's L trials, key = -ln(u(seed, round, trial, row)) / m_i over the
//             rows with m_i > 0 (an exponential race: the minimum is a draw proportional to m, independent of the
//             device split and of the launch shape)
//   reduce    one CTA: the minimum (key, row) per trial, lowest row on equal keys
//   gather    the L trial rows out of X
//   trial     the hot pass: one read of X, every row's true distance e_t to every trial row (exact.cuh's Kahan chain,
//             bit for bit), d'_t = e_t < d ? e_t : d (0 on the trial row itself), and the per-block partials of
//             phi_t = sum w d'_t^2 (block_sum)
//   pick      one CTA: phi_t folded in a fixed order (chunk_sum, fold_chunks), argmin t (lowest t on equal values), and
//             the winner row appended to C
// On one GPU every step stays on the device (GppCtl carries the winner from the pick to the next draw); with several
// GPUs the host merges the keys and the potentials between the steps.
#include <algorithm>

#include "exact.cuh"
#include "fixed_order.cuh"
#include "kernels.h"

namespace kmb {

namespace {

constexpr int kGppRows = kStagedRows;  // rows per CTA of the trial pass (= threads)
constexpr int kGppDrawThreads = 256;   // rows per tile of the draw pass
constexpr int kGppFoldGroup = 4;       // trials whose chunk sums the pick kernel holds in shared memory at once

__device__ __forceinline__ bool key_less(double ka, uint32_t ra, double kb, uint32_t rb) {
  return ka < kb || (ka == kb && ra < rb);
}

__device__ __forceinline__ void warp_min_key(double& k, uint32_t& r) {
  for (int o = 16; o > 0; o >>= 1) {
    const double ko = __shfl_down_sync(0xffffffffu, k, o);
    const uint32_t ro = __shfl_down_sync(0xffffffffu, r, o);
    if (key_less(ko, ro, k, r)) {
      k = ko;
      r = ro;
    }
  }
}

// Grid-stride over 256-row tiles.  Every row folds the winner's column into d and zeroes the chosen row, then each
// trial's (key, row) minimum of the tile is merged into the warp's running minimum in shared memory; at the end warp 0
// merges the 8 warps per trial and writes bkey / brow [L][gridDim.x].
__global__ void __launch_bounds__(kGppDrawThreads)
gpp_draw_kernel(float* __restrict__ dists, const float* __restrict__ dprime, const float* __restrict__ w, uint32_t n,
                uint32_t off, uint32_t L, const GppCtl* __restrict__ ctl, uint64_t rkey, double* __restrict__ bkey,
                uint32_t* __restrict__ brow) {
  __shared__ double s_key[kGppDrawThreads / 32][kGppMaxTrials];
  __shared__ uint32_t s_row[kGppDrawThreads / 32][kGppMaxTrials];
  if (ctl->stop) return;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const uint32_t winner = ctl->winner, chosen = ctl->chosen;
  for (uint32_t t = lane; t < L; t += 32) {
    s_key[warp][t] = INFINITY;
    s_row[warp][t] = UINT32_MAX;
  }
  __syncwarp();
  for (uint32_t base = blockIdx.x * kGppDrawThreads; base < n; base += gridDim.x * kGppDrawThreads) {
    const uint32_t i = base + threadIdx.x;
    double m = 0.0;
    if (i < n) {
      float d = winner < L ? dprime[static_cast<size_t>(winner) * n + i] : dists[i];
      if (off + i == chosen) d = 0.f;
      dists[i] = d;
      m = d2_mass(d, w ? w[i] : 1.f);
    }
    if (!__any_sync(0xffffffffu, m > 0.0)) continue;
    for (uint32_t t = 0; t < L; t++) {
      double k = INFINITY;
      uint32_t r = UINT32_MAX;
      if (m > 0.0) {
        k = -log(unit_oo(splitmix64(splitmix64(rkey + t) ^ static_cast<uint64_t>(off + i)))) / m;
        r = off + i;
      }
      warp_min_key(k, r);
      if (lane == 0 && key_less(k, r, s_key[warp][t], s_row[warp][t])) {
        s_key[warp][t] = k;
        s_row[warp][t] = r;
      }
    }
  }
  __syncthreads();
  if (warp == 0) {
    for (uint32_t t = lane; t < L; t += 32) {
      double k = s_key[0][t];
      uint32_t r = s_row[0][t];
      for (int q = 1; q < kGppDrawThreads / 32; q++)
        if (key_less(s_key[q][t], s_row[q][t], k, r)) {
          k = s_key[q][t];
          r = s_row[q][t];
        }
      bkey[static_cast<size_t>(t) * gridDim.x + blockIdx.x] = k;
      brow[static_cast<size_t>(t) * gridDim.x + blockIdx.x] = r;
    }
  }
}

// one CTA, warp t reduces trial t's nb block minima; single: no row left to draw stops the rounds
__global__ void __launch_bounds__(1024)
gpp_key_reduce_kernel(const double* __restrict__ bkey, const uint32_t* __restrict__ brow, uint32_t nb, uint32_t L,
                      GppCtl* __restrict__ ctl, double* __restrict__ keys, uint32_t* __restrict__ rows, bool single) {
  if (ctl->stop) return;
  const uint32_t lane = threadIdx.x & 31, t = threadIdx.x >> 5;
  if (t < L) {
    double k = INFINITY;
    uint32_t r = UINT32_MAX;
    for (uint32_t b = lane; b < nb; b += 32)
      if (key_less(bkey[static_cast<size_t>(t) * nb + b], brow[static_cast<size_t>(t) * nb + b], k, r)) {
        k = bkey[static_cast<size_t>(t) * nb + b];
        r = brow[static_cast<size_t>(t) * nb + b];
      }
    warp_min_key(k, r);
    if (lane == 0) {
      keys[t] = k;
      rows[t] = r;
      if (single && t == 0 && r == UINT32_MAX) ctl->stop = 1;   // phi = 0: every trial finds no row
    }
  }
}

// T[t][:] = X[rows[t] - off][:]
__global__ void gpp_gather_kernel(const float* __restrict__ X, uint32_t off, int D, const uint32_t* __restrict__ rows,
                                  uint32_t L, const GppCtl* __restrict__ ctl, float* __restrict__ T) {
  if (ctl->stop) return;
  const size_t total = static_cast<size_t>(L) * D;
  for (size_t e = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; e < total;
       e += static_cast<size_t>(gridDim.x) * blockDim.x) {
    const size_t t = e / D, f = e - t * D;
    T[e] = X[static_cast<size_t>(rows[t] - off) * D + f];
  }
}

// The trial pass.  32-feature slices of the CTA's 128 rows and of the L trial rows are staged through shared memory;
// each thread advances the L Kahan chains of its row in registers (LC >= L chains, unrolled, so that the chains of one
// feature are independent instructions).
template <int METRIC, int LC>
__global__ void __launch_bounds__(kGppRows)
gpp_trial_kernel(const float* __restrict__ X, uint32_t n, uint32_t off, int D, const float* __restrict__ T, uint32_t L,
                 const uint32_t* __restrict__ trial_rows, const float* __restrict__ dists, const float* __restrict__ w,
                 const GppCtl* __restrict__ ctl, float* __restrict__ dprime, double* __restrict__ bsum) {
  __shared__ float tile[kGppRows * 33];
  __shared__ __align__(16) float s_t[LC * 32];
  __shared__ double s_part[kGppRows / 32];
  if (ctl->stop) return;
  const int t = threadIdx.x;
  const uint32_t row0 = blockIdx.x * kGppRows, i = row0 + t;
  const bool live = i < n;
  Kahan k[LC];
  for (int f0 = 0; f0 < D; f0 += 32) {
    const int fl = min(32, D - f0);
    stage_slice(X, RowRange{row0}, row0, n, D, f0, fl, tile);
    for (uint32_t e = t; e < L * 32; e += kGppRows) {
      const uint32_t q = e >> 5, f = e & 31;
      s_t[e] = static_cast<int>(f) < fl ? T[static_cast<size_t>(q) * D + f0 + f] : 0.f;
    }
    __syncthreads();
    if (live) {
      const float* xs = tile + t * 33;
      if (fl == 32) {
#pragma unroll 1
        for (int v = 0; v < 8; v++) {
          const float x0 = xs[4 * v], x1 = xs[4 * v + 1], x2 = xs[4 * v + 2], x3 = xs[4 * v + 3];
#pragma unroll
          for (int q = 0; q < LC; q++) {
            if (q < static_cast<int>(L)) {
              const float4 c = reinterpret_cast<const float4*>(s_t + q * 32)[v];
              if (METRIC == 1) {
                k[q].mac(x0, c.x); k[q].mac(x1, c.y); k[q].mac(x2, c.z); k[q].mac(x3, c.w);
              } else {
                k[q].sqdiff(x0, c.x); k[q].sqdiff(x1, c.y); k[q].sqdiff(x2, c.z); k[q].sqdiff(x3, c.w);
              }
            }
          }
        }
      } else {
        for (int f = 0; f < fl; f++) {
#pragma unroll
          for (int q = 0; q < LC; q++) {
            if (q < static_cast<int>(L)) {
              if (METRIC == 1) k[q].mac(xs[f], s_t[q * 32 + f]);
              else k[q].sqdiff(xs[f], s_t[q * 32 + f]);
            }
          }
        }
      }
    }
    __syncthreads();
  }
  float d = 0.f, wi = 1.f;
  bool nan_row = false;
  if (live) {
    d = dists[i];
    if (w) wi = w[i];
    nan_row = !(X[static_cast<size_t>(i) * D] == X[static_cast<size_t>(i) * D]);
  }
  const uint32_t nb = gridDim.x;
#pragma unroll
  for (int q = 0; q < LC; q++) {
    if (q < static_cast<int>(L)) {
      double m = 0.0;
      if (live) {
        float dp = d;
        if (off + i == trial_rows[q]) {
          dp = 0.f;
        } else if (!nan_row) {
          const float e = finalize_distance<METRIC>(k[q].sum);
          if (e < d) dp = e;
        }
        dprime[static_cast<size_t>(q) * n + i] = dp;
        m = d2_mass(dp, wi);
      }
      const double s = block_sum<kGppRows>(m, s_part);
      if (t == 0) bsum[static_cast<size_t>(q) * nb + blockIdx.x] = s;
      __syncthreads();
    }
  }
}

template <int METRIC>
void gpp_trial_dispatch(const float* X, uint32_t n, uint32_t off, int D, const float* T, uint32_t L,
                        const uint32_t* trial_rows, const float* dists, const float* w, const GppCtl* ctl,
                        float* dprime, double* bsum, cudaStream_t st) {
  const unsigned grid = cdiv(n, kGppRows);
  if (L <= 2)
    gpp_trial_kernel<METRIC, 2><<<grid, kGppRows, 0, st>>>(X, n, off, D, T, L, trial_rows, dists, w, ctl, dprime, bsum);
  else if (L <= 4)
    gpp_trial_kernel<METRIC, 4><<<grid, kGppRows, 0, st>>>(X, n, off, D, T, L, trial_rows, dists, w, ctl, dprime, bsum);
  else if (L <= 8)
    gpp_trial_kernel<METRIC, 8><<<grid, kGppRows, 0, st>>>(X, n, off, D, T, L, trial_rows, dists, w, ctl, dprime, bsum);
  else if (L <= 16)
    gpp_trial_kernel<METRIC, 16><<<grid, kGppRows, 0, st>>>(X, n, off, D, T, L, trial_rows, dists, w, ctl, dprime, bsum);
  else
    gpp_trial_kernel<METRIC, 32><<<grid, kGppRows, 0, st>>>(X, n, off, D, T, L, trial_rows, dists, w, ctl, dprime, bsum);
}

// One CTA: phis[t] = trial t's block partials folded in a fixed order (chunk_sum, fold_chunks).  pick: thread 0 takes
// the argmin t (lowest t on equal values), records it in ctl and the round log, and the CTA copies the winner row into
// crow.
__global__ void __launch_bounds__(1024)
gpp_pick_kernel(const double* __restrict__ bsum, uint32_t nb, uint32_t L, GppCtl* __restrict__ ctl,
                const uint32_t* __restrict__ trial_rows, double* __restrict__ phis, bool pick,
                const float* __restrict__ X, uint32_t off, int D, float* __restrict__ crow,
                uint32_t* __restrict__ row_log, double* __restrict__ phi_log) {
  __shared__ double s_chunk[kGppFoldGroup][1024];
  __shared__ uint32_t s_chosen;
  if (ctl->stop) return;
  for (uint32_t t0 = 0; t0 < L; t0 += kGppFoldGroup) {
    for (uint32_t g = 0; g < kGppFoldGroup && t0 + g < L; g++)
      s_chunk[g][threadIdx.x] = chunk_sum(bsum + static_cast<size_t>(t0 + g) * nb, nb);
    __syncthreads();
    if (threadIdx.x < kGppFoldGroup && t0 + threadIdx.x < L) phis[t0 + threadIdx.x] = fold_chunks(s_chunk[threadIdx.x]);
    __syncthreads();
  }
  if (!pick) return;
  if (threadIdx.x == 0) {
    uint32_t best = 0;
    for (uint32_t t = 1; t < L; t++)
      if (phis[t] < phis[best]) best = t;
    ctl->winner = best;
    ctl->chosen = trial_rows[best];
    *row_log = trial_rows[best];
    *phi_log = phis[best];
    s_chosen = trial_rows[best];
  }
  __syncthreads();
  const float* x = X + static_cast<size_t>(s_chosen - off) * D;
  for (int f = threadIdx.x; f < D; f += blockDim.x) crow[f] = x[f];
}

}  // namespace

uint64_t gpp_round_key(uint32_t seed, uint32_t round) { return mb_step_key(seed, round, kGppTagTrial); }

uint32_t gpp_draw_blocks(uint32_t n) { return std::max(1u, std::min(cdiv(n, kGppDrawThreads), device_sms() * 4u)); }

uint32_t gpp_trial_blocks(uint32_t n) { return std::max(1u, cdiv(n, kGppRows)); }

cudaError_t launch_gpp_draw(float* dists, const float* dprime, const float* w, uint32_t n, uint32_t off, uint32_t L,
                            const GppCtl* ctl, uint64_t rkey, double* bkey, uint32_t* brow, double* keys,
                            uint32_t* rows, GppCtl* ctl_w, bool single, cudaStream_t st) {
  const uint32_t nb = gpp_draw_blocks(n);
  if (n > 0) {
    gpp_draw_kernel<<<nb, kGppDrawThreads, 0, st>>>(dists, dprime, w, n, off, L, ctl, rkey, bkey, brow);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return e;
  }
  gpp_key_reduce_kernel<<<1, 1024, 0, st>>>(bkey, brow, n > 0 ? nb : 0, L, ctl_w, keys, rows, single);
  return cudaGetLastError();
}

cudaError_t launch_gpp_gather(const float* X, uint32_t off, int D, const uint32_t* rows, uint32_t L, const GppCtl* ctl,
                              float* T, cudaStream_t st) {
  const size_t total = static_cast<size_t>(L) * D;
  gpp_gather_kernel<<<std::min<size_t>(cdiv(total, 256), device_sms() * 8u), 256, 0, st>>>(X, off, D, rows, L, ctl, T);
  return cudaGetLastError();
}

cudaError_t launch_gpp_trial(int metric, const float* X, uint32_t n, uint32_t off, int D, const float* T, uint32_t L,
                             const uint32_t* trial_rows, const float* dists, const float* w, const GppCtl* ctl,
                             float* dprime, double* bsum, cudaStream_t st) {
  if (n == 0) return cudaMemsetAsync(bsum, 0, sizeof(double) * L, st);
  if (metric == 1) gpp_trial_dispatch<1>(X, n, off, D, T, L, trial_rows, dists, w, ctl, dprime, bsum, st);
  else gpp_trial_dispatch<0>(X, n, off, D, T, L, trial_rows, dists, w, ctl, dprime, bsum, st);
  return cudaGetLastError();
}

cudaError_t launch_gpp_pick(const double* bsum, uint32_t n, uint32_t L, GppCtl* ctl, const uint32_t* trial_rows,
                            double* phis, bool pick, const float* X, uint32_t off, int D, float* crow,
                            uint32_t* row_log, double* phi_log, cudaStream_t st) {
  gpp_pick_kernel<<<1, 1024, 0, st>>>(bsum, gpp_trial_blocks(n), L, ctl, trial_rows, phis, pick, X, off, D, crow,
                                      row_log, phi_log);
  return cudaGetLastError();
}

}  // namespace kmb
