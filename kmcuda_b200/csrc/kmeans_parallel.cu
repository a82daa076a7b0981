// kmeans_parallel.cu -- device side of the k-means|| seeding (Bahmani et al., "Scalable K-Means++", VLDB 2012).
//
// A round of the seeding (Job::init_kmeans_parallel, seeding.cu) is
//   draw      every row i is drawn iff u(seed, r, i) < l * w_i d_i^2 / phi, u a stateless counter hash of the global
//             row index, so the draws do not depend on the device split or the launch shape; the drawn local row ids
//             are compacted in ascending order (cub::DeviceSelect::Flagged) and their rows gathered
//   assign    one assignment pass of the shard against the round's new candidates (Shard::assign, not here)
//   update    d_i = min(d_i, true distance to the pass's winner), nearest_i = its list index, and the per-block partials
//             of the next round's phi = sum w_i d_i^2 (one double per block, fixed order, no atomics)
// and at the end the candidate weights W_j = sum of w_i over nearest_i == j are reduced deterministically.
//
// The update kernel is a streaming pass over the samples (D * 4 + ~16 bytes per row): 32-feature slices of 128 rows
// are staged through padded shared memory with coalesced loads, then every thread advances the sequential Kahan chain
// of its own row (exact.cuh's distance_exact, bit for bit) over the slice.
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_select.cuh>
#include <thrust/iterator/counting_iterator.h>

#include <algorithm>

#include "exact.cuh"
#include "fixed_order.cuh"
#include "kernels.h"

namespace kmb {

namespace {

constexpr int kKmpRows = kStagedRows;   // rows per CTA of the update kernel (= threads)

// FIRST: the distance to c0 (cand, one row) starts every row's running minimum, nearest = 0.  Otherwise: the true
// distance e to the round's winner cand[assign[i]] replaces d_i when e < d_i, nearest_i = base + assign[i].
// Rows whose first feature is NaN keep d = 0 (pp_update_kernel's rule).  VEC4: D % 4 == 0, candidate rows read as float4.
template <int METRIC, bool FIRST, bool VEC4>
__global__ void __launch_bounds__(kKmpRows)
kmp_update_kernel(const float* __restrict__ X, uint32_t n, int D, const float* __restrict__ cand, uint32_t ncand,
                  const uint32_t* __restrict__ assign, uint32_t base, float* __restrict__ dists,
                  uint32_t* __restrict__ nearest, const float* __restrict__ w, double* __restrict__ bsum) {
  __shared__ float tile[kKmpRows * 33];
  __shared__ double s_part[kKmpRows / 32];
  const uint32_t row0 = blockIdx.x * kKmpRows, i = row0 + threadIdx.x;
  uint32_t a = 0;
  if (!FIRST && i < n) a = assign[i];
  const bool live = i < n && (FIRST || a < ncand);
  const float* c = cand + static_cast<size_t>(live ? a : 0) * D;
  const float sum = staged_own_sum<VEC4, METRIC>(X, RowRange{row0}, row0, n, D, c, live, tile);
  double m = 0.0;
  if (i < n) {
    const bool nan_row = !(X[static_cast<size_t>(i) * D] == X[static_cast<size_t>(i) * D]);
    float d;
    if (FIRST) {
      d = nan_row ? 0.f : finalize_distance<METRIC>(sum);
      dists[i] = d;
      nearest[i] = 0;
    } else {
      d = dists[i];
      if (live && !nan_row) {
        const float e = finalize_distance<METRIC>(sum);
        if (e < d) {
          d = e;
          dists[i] = e;
          nearest[i] = base + a;
        }
      }
    }
    m = d2_mass(d, w ? w[i] : 1.f);
  }
  const double s = block_sum<kKmpRows>(m, s_part);
  if (threadIdx.x == 0) bsum[blockIdx.x] = s;
}

__global__ void kmp_flag_kernel(const float* __restrict__ dists, const float* __restrict__ w, uint32_t n, uint32_t off,
                                uint64_t key, double ell, double phi, uint8_t* __restrict__ flags) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const double u = unit_co(splitmix64(key ^ static_cast<uint64_t>(off + i)));
  const double m = d2_mass(dists[i], w ? w[i] : 1.f);
  flags[i] = u < (ell * m) / phi;
}

__global__ void kmp_gather_kernel(const float* __restrict__ X, int D, const uint32_t* __restrict__ idx, uint32_t cnt,
                                  float* __restrict__ out) {
  const size_t total = static_cast<size_t>(cnt) * D;
  for (size_t e = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; e < total;
       e += static_cast<size_t>(gridDim.x) * blockDim.x) {
    const size_t j = e / D, f = e - j * D;
    out[e] = X[static_cast<size_t>(idx[j]) * D + f];
  }
}

__global__ void kmp_count_kernel(const uint32_t* __restrict__ nearest, uint32_t n, uint32_t* __restrict__ counts) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) atomicAdd(counts + nearest[i], 1u);
}

// run bounds of the sorted keys: start[k] = first position of key k, start[C + k] = one past its last (both pre-filled
// with n, so an absent key is the empty run [n, n))
__global__ void kmp_run_bounds_kernel(const uint32_t* __restrict__ keys, uint32_t n, uint32_t C,
                                      uint32_t* __restrict__ start) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  if (i == 0 || keys[i] != keys[i - 1]) start[keys[i]] = i;
  if (i == n - 1 || keys[i + 1] != keys[i]) start[C + keys[i]] = i + 1;
}

constexpr int kRunThreads = 256;

__device__ __forceinline__ void kahan_add(float& s, float& corr, float v) {
  const float y = v - corr;
  const float t = s + y;
  corr = (t - s) - y;
  s = t;
}

// W[j] = compensated sum of the weights of run j, one CTA per run: thread t sums positions start + t, start + t + 256,
// ... in row order (the sort is stable), then thread 0 adds the 256 partials in thread order.  The order depends only
// on the run, so the total is deterministic, and a skewed run (most rows nearest to one candidate) is spread over the
// CTA instead of one thread.
__global__ void __launch_bounds__(kRunThreads)
kmp_run_sums_kernel(const float* __restrict__ vals, const uint32_t* __restrict__ start, uint32_t C,
                    float* __restrict__ W) {
  __shared__ float s_part[kRunThreads];
  const uint32_t j = blockIdx.x, lo = start[j], hi = start[C + j];
  float s = 0.f, corr = 0.f;
  for (uint32_t i = lo + threadIdx.x; i < hi; i += kRunThreads) kahan_add(s, corr, vals[i]);
  s_part[threadIdx.x] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    float t = 0.f, c = 0.f;
    for (int q = 0; q < kRunThreads; q++) kahan_add(t, c, s_part[q]);
    W[j] = t;
  }
}

template <int METRIC, bool FIRST>
void kmp_update_dispatch(const float* X, uint32_t n, int D, const float* cand, uint32_t ncand, const uint32_t* assign,
                         uint32_t base, float* dists, uint32_t* nearest, const float* w, double* bsum, cudaStream_t st) {
  const unsigned grid = cdiv(n, kKmpRows);
  if (D % 4 == 0)
    kmp_update_kernel<METRIC, FIRST, true><<<grid, kKmpRows, 0, st>>>(X, n, D, cand, ncand, assign, base, dists,
                                                                       nearest, w, bsum);
  else
    kmp_update_kernel<METRIC, FIRST, false><<<grid, kKmpRows, 0, st>>>(X, n, D, cand, ncand, assign, base, dists,
                                                                        nearest, w, bsum);
}

}  // namespace

uint32_t kmp_blocks(uint32_t n) { return std::max(1u, cdiv(n, kKmpRows)); }

cudaError_t launch_kmp_update(int metric, const float* X, uint32_t n, int D, const float* cand, uint32_t ncand,
                              const uint32_t* assign, uint32_t base, float* dists, uint32_t* nearest, const float* w,
                              double* bsum, cudaStream_t st) {
  if (n == 0) return cudaMemsetAsync(bsum, 0, sizeof(double), st);
  const bool first = assign == nullptr;
  if (metric == 1) {
    if (first) kmp_update_dispatch<1, true>(X, n, D, cand, ncand, assign, base, dists, nearest, w, bsum, st);
    else kmp_update_dispatch<1, false>(X, n, D, cand, ncand, assign, base, dists, nearest, w, bsum, st);
  } else {
    if (first) kmp_update_dispatch<0, true>(X, n, D, cand, ncand, assign, base, dists, nearest, w, bsum, st);
    else kmp_update_dispatch<0, false>(X, n, D, cand, ncand, assign, base, dists, nearest, w, bsum, st);
  }
  return cudaGetLastError();
}

size_t kmp_select_bytes(uint32_t n) {
  size_t bytes = 0;
  thrust::counting_iterator<uint32_t> it(0);
  cub::DeviceSelect::Flagged(nullptr, bytes, it, static_cast<const uint8_t*>(nullptr), static_cast<uint32_t*>(nullptr),
                             static_cast<uint32_t*>(nullptr), std::max(n, 1u));
  return bytes;
}

cudaError_t launch_kmp_draw(const float* dists, const float* w, uint32_t n, uint32_t off, uint32_t seed, uint32_t round,
                            double ell, double phi, uint8_t* flags, uint32_t* idx, uint32_t* d_count, void* tmp,
                            size_t tmp_bytes, cudaStream_t st) {
  if (n == 0) return cudaMemsetAsync(d_count, 0, sizeof(uint32_t), st);
  const uint64_t key = splitmix64((static_cast<uint64_t>(seed) << 8) | round);
  kmp_flag_kernel<<<cdiv(n, 256), 256, 0, st>>>(dists, w, n, off, key, ell, phi, flags);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return e;
  thrust::counting_iterator<uint32_t> it(0);
  return cub::DeviceSelect::Flagged(tmp, tmp_bytes, it, flags, idx, d_count, n, st);
}

cudaError_t launch_kmp_gather(const float* X, int D, const uint32_t* idx, uint32_t cnt, float* out, cudaStream_t st) {
  if (cnt == 0) return cudaSuccess;
  const size_t total = static_cast<size_t>(cnt) * D;
  kmp_gather_kernel<<<std::min<size_t>(cdiv(total, 256), device_sms() * 8u), 256, 0, st>>>(X, D, idx, cnt, out);
  return cudaGetLastError();
}

cudaError_t launch_kmp_counts(const uint32_t* nearest, uint32_t n, uint32_t* counts, cudaStream_t st) {
  if (n == 0) return cudaSuccess;
  kmp_count_kernel<<<cdiv(n, 256), 256, 0, st>>>(nearest, n, counts);
  return cudaGetLastError();
}

size_t kmp_weights_bytes(uint32_t n) {
  size_t bytes = 0;
  cub::DeviceRadixSort::SortPairs(nullptr, bytes, static_cast<const uint32_t*>(nullptr),
                                  static_cast<uint32_t*>(nullptr), static_cast<const float*>(nullptr),
                                  static_cast<float*>(nullptr), std::max(n, 1u));
  return bytes;
}

cudaError_t launch_kmp_weights(const uint32_t* nearest, const float* w, uint32_t n, uint32_t C, uint32_t* keys_out,
                               float* w_out, uint32_t* start, void* tmp, size_t tmp_bytes, float* W, cudaStream_t st) {
  cudaError_t e = launch_fill_u32(start, n, 2 * static_cast<size_t>(C), st);
  if (e != cudaSuccess) return e;
  if (n > 0) {
    int end_bit = 1;
    while (end_bit < 32 && (C - 1) >> end_bit) end_bit++;
    e = cub::DeviceRadixSort::SortPairs(tmp, tmp_bytes, nearest, keys_out, w, w_out, n, 0, end_bit, st);
    if (e != cudaSuccess) return e;
    kmp_run_bounds_kernel<<<cdiv(n, 256), 256, 0, st>>>(keys_out, n, C, start);
  }
  kmp_run_sums_kernel<<<C, kRunThreads, 0, st>>>(w_out, start, C, W);
  return cudaGetLastError();
}

}  // namespace kmb
