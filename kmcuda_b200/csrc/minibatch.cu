// minibatch.cu -- device side of mini-batch k-means (Sculley, "Web-scale k-means clustering", WWW 2010; the update and
// reassignment rules of scikit-learn's MiniBatchKMeans).  A step of Job::minibatch (job.cu) is
//   draw       row_j = floor(u(seed, s, j) * N) for the b batch entries j (with replacement), w_j = w[row_j]; u is a
//              SplitMix64 counter hash with its own domain tag, so the draws depend on (seed, s, j) only
//   assign     Shard::assign_rows: the exact argmin of every entry, the tensor-core pass reading X[row_j] itself
//   inertia    sum_j w_j ||X[row_j] - c_{a_j}||^2 (the reference's L2 Kahan sum before its square root), block partials
//              in double added in a fixed order (launch_fixed_sum)
//   sums       the existing deterministic member sums (launch_partial_sums) with the entries' rows as the sorted values
//   blend      c <- (c W_c + S_c) / (W_c + W_b,c), W_c += W_b,c for every centroid with W_b,c > 0
//   reassign   (when the host says so) the centroids with W_c < 0.01 max W, at most floor(b / 2) of the smallest, become
//              batch entries drawn proportionally to w_j without replacement (Efraimidis-Spirakis keys -log(u) / w_j)
//   stats      sum_c ||c_new - c_old||^2 and the number of centroids with W_c == 0, for the host's stop decision
#include <cub/device/device_radix_sort.cuh>

#include <algorithm>
#include <cmath>

#include "exact.cuh"
#include "fixed_order.cuh"
#include "kernels.h"

namespace kmb {

namespace {

constexpr int kMbRows = kStagedRows;   // rows per CTA of the inertia kernel (= threads)

__global__ void mb_draw_kernel(uint32_t N, uint32_t b, uint64_t key, uint32_t* __restrict__ rows) {
  const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= b) return;
  rows[j] = min(static_cast<uint32_t>(unit_co(splitmix64(key ^ j)) * N), N - 1);
}

// Exact squared L2 distance of every entry to its centroid (staged_own_sum).  Entries whose winner is not a centroid
// (K for a NaN row, kUntouched when every score is NaN) carry no inertia and are given the key K, so the member sums
// skip them.
template <bool VEC4>
__global__ void __launch_bounds__(kMbRows)
mb_inertia_kernel(const float* __restrict__ X, const uint32_t* __restrict__ rows, uint32_t n, int D,
                  const float* __restrict__ C, uint32_t K, const uint32_t* __restrict__ result,
                  const float* __restrict__ w, uint32_t* __restrict__ keys, double* __restrict__ bsum) {
  __shared__ uint32_t s_row[kMbRows];
  __shared__ float tile[kMbRows * 33];
  __shared__ double s_part[kMbRows / 32];
  const int t = threadIdx.x;
  const uint32_t row0 = blockIdx.x * kMbRows, i = row0 + t;
  uint32_t a = K;
  if (i < n) a = min(result[i], K);
  const bool live = a < K;
  const float* c = C + static_cast<size_t>(live ? a : 0) * D;
  s_row[t] = i < n ? rows[i] : 0u;
  __syncthreads();
  const float sum = staged_own_sum<VEC4, 0>(X, s_row, row0, n, D, c, live, tile);
  double m = 0.0;
  if (i < n) {
    keys[i] = a;
    if (live) m = static_cast<double>(w ? w[s_row[t]] : 1.f) * static_cast<double>(sum);
  }
  const double s = block_sum<kMbRows>(m, s_part);
  if (t == 0) bsum[blockIdx.x] = s;
}

// c_new = (c W + S) / (W + W_b) where W_b > 0, else c; W_new = W + W_b
__global__ void mb_blend_kernel(const float* __restrict__ C, const double* __restrict__ W, const float* __restrict__ S,
                                const float* __restrict__ wsums, const uint32_t* __restrict__ counts, uint32_t K,
                                int D, float* __restrict__ Cnew, double* __restrict__ Wnew) {
  const size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= static_cast<size_t>(K) * D) return;
  const uint32_t c = i / D;
  const double wb = wsums ? static_cast<double>(wsums[c]) : static_cast<double>(static_cast<float>(counts[c]));
  const double w = W[c];
  Cnew[i] = wb > 0 ? static_cast<float>((static_cast<double>(C[i]) * w + static_cast<double>(S[i])) / (w + wb)) : C[i];
  if (i - static_cast<size_t>(c) * D == 0) Wnew[c] = w + wb;
}

// Efraimidis-Spirakis key of every batch entry: -log(u) / w_j (the smallest keys are the draw), +inf for w_j = 0;
// *npos += entries of positive weight
__global__ void mb_reassign_keys_kernel(uint32_t b, uint64_t key, const float* __restrict__ wrow,
                                        const uint32_t* __restrict__ rows, double* __restrict__ ekey,
                                        uint32_t* __restrict__ pos, uint32_t* npos) {
  const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= b) return;
  const float w = wrow ? wrow[rows[j]] : 1.f;
  ekey[j] = w > 0.f ? -log(unit_oo(splitmix64(key ^ j))) / static_cast<double>(w) : INFINITY;
  pos[j] = j;
  const unsigned act = __activemask();
  const unsigned live = __ballot_sync(act, w > 0.f);
  if ((threadIdx.x & 31) == __ffs(act) - 1 && live) atomicAdd(npos, static_cast<uint32_t>(__popc(live)));
}

__global__ void mb_iota_kernel(uint32_t* __restrict__ p, uint32_t n) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) p[i] = i;
}

// Wsorted ascending (stable): m = min(#{W < ratio * max W}, floor(b / 2), npos); out[0] = m, out[1] = the smallest kept W
__global__ void mb_reassign_pick_kernel(const double* __restrict__ Wsorted, uint32_t K, uint32_t half_b,
                                        const uint32_t* __restrict__ npos, double ratio, uint32_t* __restrict__ m_out,
                                        double* __restrict__ minkept) {
  const double thr = ratio * Wsorted[K - 1];
  uint32_t lo = 0, hi = K;   // lower_bound(thr)
  while (lo < hi) {
    const uint32_t mid = (lo + hi) / 2;
    if (Wsorted[mid] < thr) lo = mid + 1;
    else hi = mid;
  }
  const uint32_t m = min(min(lo, half_b), *npos);
  *m_out = m;
  *minkept = m < K ? Wsorted[m] : Wsorted[K - 1];
}

// the r-th smallest W (stable order) takes the r-th drawn entry, r < m; its W becomes the smallest kept W
__global__ void mb_reassign_apply_kernel(const uint32_t* __restrict__ cidx, const uint32_t* __restrict__ picked,
                                         const uint32_t* __restrict__ m_in, const double* __restrict__ minkept,
                                         const float* __restrict__ X, const uint32_t* __restrict__ rows, int D,
                                         uint32_t rmax, float* __restrict__ C, double* __restrict__ W) {
  const size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= static_cast<size_t>(rmax) * D) return;
  const uint32_t r = i / D;
  if (r >= *m_in) return;
  const int f = static_cast<int>(i - static_cast<size_t>(r) * D);
  const uint32_t c = cidx[r];
  C[static_cast<size_t>(c) * D + f] = X[static_cast<size_t>(rows[picked[r]]) * D + f];
  if (f == 0) W[c] = *minkept;
}

// dsq[c] = ||Cnew_c - Cold_c||^2 in double, one CTA per centroid, fixed reduction order
__global__ void __launch_bounds__(128)
mb_shift_kernel(const float* __restrict__ Cold, const float* __restrict__ Cnew, int D, double* __restrict__ dsq) {
  __shared__ double s_part[4];
  const uint32_t c = blockIdx.x;
  double acc = 0.0;
  for (int f = threadIdx.x; f < D; f += 128) {
    const double d = static_cast<double>(Cnew[static_cast<size_t>(c) * D + f]) - Cold[static_cast<size_t>(c) * D + f];
    acc += d * d;
  }
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_down_sync(0xffffffffu, acc, o);
  if ((threadIdx.x & 31) == 0) s_part[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) dsq[c] = ((s_part[0] + s_part[1]) + s_part[2]) + s_part[3];
}

// out[0] = sum of dsq[K] (chunk_sum, fold_chunks), out[1] = #{W_c == 0}
__global__ void __launch_bounds__(1024)
mb_stats_kernel(const double* __restrict__ dsq, const double* __restrict__ W, uint32_t K, double* __restrict__ out) {
  __shared__ double s_chunk[1024];
  __shared__ uint32_t s_zero;
  if (threadIdx.x == 0) s_zero = 0;
  __syncthreads();
  s_chunk[threadIdx.x] = chunk_sum(dsq, K);
  uint32_t lo, hi, z = 0;
  chunk_range(K, lo, hi);
  for (uint32_t c = lo; c < hi; c++) z += W[c] == 0.0;
  if (z) atomicAdd(&s_zero, z);
  __syncthreads();
  if (threadIdx.x == 0) {
    out[0] = fold_chunks(s_chunk);
    out[1] = static_cast<double>(s_zero);
  }
}

// out[0] = sum of dsq[K] with the non-finite terms as 0 (chunk_sum, fold_chunks): the centre shift of a Lloyd / Yinyang
// update under scikit-learn's stopping rule, where a dead centroid (NaN) must not keep a run going
__global__ void __launch_bounds__(1024)
center_shift_fold_kernel(const double* __restrict__ dsq, uint32_t K, double* __restrict__ out) {
  __shared__ double s_chunk[1024];
  s_chunk[threadIdx.x] = chunk_sum<true>(dsq, K);
  __syncthreads();
  if (threadIdx.x == 0) out[0] = fold_chunks(s_chunk);
}

// per-feature variance, two passes in double: partial[b][f] over a contiguous row range per CTA, folded in CTA order
constexpr int kVarBlocks = 256;
__global__ void __launch_bounds__(256)
mb_colsum_kernel(const float* __restrict__ X, uint32_t n, int D, const double* __restrict__ mean,
                 double* __restrict__ partial) {
  const uint32_t per = (n + gridDim.x - 1) / gridDim.x;
  const uint32_t lo = min(n, blockIdx.x * per), hi = min(n, lo + per);
  for (int f = threadIdx.x; f < D; f += blockDim.x) {
    double acc = 0.0;
    const double m = mean ? mean[f] : 0.0;
#pragma unroll 8
    for (uint32_t r = lo; r < hi; r++) {
      const double v = static_cast<double>(X[static_cast<size_t>(r) * D + f]) - m;
      acc += mean ? v * v : v;
    }
    partial[static_cast<size_t>(blockIdx.x) * D + f] = acc;
  }
}

__global__ void mb_colfold_kernel(const double* __restrict__ partial, int nb, int D, double* __restrict__ out) {
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= D) return;
  double acc = 0.0;
  for (int q = 0; q < nb; q++) acc += partial[static_cast<size_t>(q) * D + f];
  out[f] = acc;
}

}  // namespace

uint64_t mb_step_key(uint32_t seed, uint64_t step, uint64_t tag) { return splitmix64(splitmix64(tag ^ seed) + step); }

cudaError_t launch_mb_draw(uint32_t N, uint32_t b, uint64_t key, uint32_t* rows, cudaStream_t st) {
  if (b == 0) return cudaSuccess;
  mb_draw_kernel<<<cdiv(b, 256), 256, 0, st>>>(N, b, key, rows);
  return cudaGetLastError();
}

uint32_t mb_blocks(uint32_t n) { return std::max(1u, cdiv(n, kMbRows)); }

cudaError_t launch_mb_inertia(const float* X, const uint32_t* rows, uint32_t n, int D, const float* C, uint32_t K,
                              const uint32_t* result, const float* w, uint32_t* keys, double* bsum, cudaStream_t st) {
  if (n == 0) return cudaMemsetAsync(bsum, 0, sizeof(double), st);
  if (D % 4 == 0)
    mb_inertia_kernel<true><<<cdiv(n, kMbRows), kMbRows, 0, st>>>(X, rows, n, D, C, K, result, w, keys, bsum);
  else
    mb_inertia_kernel<false><<<cdiv(n, kMbRows), kMbRows, 0, st>>>(X, rows, n, D, C, K, result, w, keys, bsum);
  return cudaGetLastError();
}

cudaError_t launch_mb_blend(const float* C, const double* W, const float* S, const float* wsums,
                            const uint32_t* counts, uint32_t K, int D, float* Cnew, double* Wnew, cudaStream_t st) {
  mb_blend_kernel<<<cdiv(static_cast<size_t>(K) * D, 256), 256, 0, st>>>(C, W, S, wsums, counts, K, D, Cnew, Wnew);
  return cudaGetLastError();
}

size_t mb_reassign_bytes(uint32_t b, uint32_t K) {
  size_t b1 = 0, b2 = 0;
  cub::DeviceRadixSort::SortPairs(nullptr, b1, static_cast<const double*>(nullptr), static_cast<double*>(nullptr),
                                  static_cast<const uint32_t*>(nullptr), static_cast<uint32_t*>(nullptr),
                                  std::max(b, 1u));
  cub::DeviceRadixSort::SortPairs(nullptr, b2, static_cast<const double*>(nullptr), static_cast<double*>(nullptr),
                                  static_cast<const uint32_t*>(nullptr), static_cast<uint32_t*>(nullptr),
                                  std::max(K, 1u));
  return std::max(b1, b2);
}

cudaError_t launch_mb_reassign(const MbReassign& r, cudaStream_t st) {
  cudaError_t e;
  // the centroids by W, ascending and stable (the identity permutation goes in as the values)
  mb_iota_kernel<<<cdiv(r.K, 256), 256, 0, st>>>(r.cidx_in, r.K);
  size_t bytes = r.tmp_bytes;
  if ((e = cub::DeviceRadixSort::SortPairs(r.tmp, bytes, r.W, r.wsorted, r.cidx_in, r.cidx, r.K, 0, 64, st)) !=
      cudaSuccess)
    return e;
  // the entries by key, ascending and stable
  if ((e = cudaMemsetAsync(r.npos, 0, sizeof(uint32_t), st)) != cudaSuccess) return e;
  mb_reassign_keys_kernel<<<cdiv(r.b, 256), 256, 0, st>>>(r.b, r.key, r.w, r.rows, r.ekey_in, r.pos_in, r.npos);
  if ((e = cudaGetLastError()) != cudaSuccess) return e;
  bytes = r.tmp_bytes;
  if ((e = cub::DeviceRadixSort::SortPairs(r.tmp, bytes, r.ekey_in, r.ekey, r.pos_in, r.picked, r.b, 0, 64, st)) !=
      cudaSuccess)
    return e;
  mb_reassign_pick_kernel<<<1, 1, 0, st>>>(r.wsorted, r.K, r.b / 2, r.npos, r.ratio, r.m, r.minkept);
  const uint32_t rmax = std::min(r.K, r.b / 2);
  if (rmax > 0)
    mb_reassign_apply_kernel<<<cdiv(static_cast<size_t>(rmax) * r.D, 256), 256, 0, st>>>(
        r.cidx, r.picked, r.m, r.minkept, r.X, r.rows, r.D, rmax, r.C, r.W);
  return cudaGetLastError();
}

cudaError_t launch_mb_stats(const float* Cold, const float* Cnew, const double* W, uint32_t K, int D, double* dsq,
                            double* out, cudaStream_t st) {
  mb_shift_kernel<<<K, 128, 0, st>>>(Cold, Cnew, D, dsq);
  mb_stats_kernel<<<1, 1024, 0, st>>>(dsq, W, K, out);
  return cudaGetLastError();
}

cudaError_t launch_center_shift(const float* Cold, const float* Cnew, uint32_t K, int D, double* dsq, double* out,
                                cudaStream_t st) {
  mb_shift_kernel<<<K, 128, 0, st>>>(Cold, Cnew, D, dsq);
  center_shift_fold_kernel<<<1, 1024, 0, st>>>(dsq, K, out);
  return cudaGetLastError();
}

size_t col_sums_doubles(int D) { return static_cast<size_t>(kVarBlocks) * D; }

cudaError_t launch_col_sums(const float* X, uint32_t n, int D, const double* mean, double* work, double* out,
                            cudaStream_t st) {
  mb_colsum_kernel<<<kVarBlocks, 256, 0, st>>>(X, n, D, mean, work);
  mb_colfold_kernel<<<cdiv(D, 256), 256, 0, st>>>(work, kVarBlocks, D, out);
  return cudaGetLastError();
}

}  // namespace kmb
