// knn_kernels.cu -- exact parts of the cluster-pruned k-NN (reference knn.cu:19-347), row-major samples: cluster radii,
// centroid distance matrix, and the warp-per-query exact search that serves whatever the tensor-core candidate pass
// (assign_tc.cu MODE 2) does not.  Decision arithmetic = the reference's: true distances by Kahan-compensated
// round-down FMA sums (exact.cuh), cluster skip test `Cd[B][A] - d(q,A) - R[B] > kth` (knn.cu:218-225), candidates
// enter on `dist <= kth`, neighbours come out in ascending distance order.
#include <algorithm>

#include "exact.cuh"
#include "kernels.h"

namespace kmb {

// distance accumulated over feature chunks: fresh Kahan sum per chunk, chunks added with a plain
// fp32 add, finalize at the end (knn.cu:36-47 with 16-feature chunks, knn.cu:79-100 with 24)
template <int METRIC, int CHUNK>
__device__ __forceinline__ float chunked_distance(const float* __restrict__ a,
                                                  const float* __restrict__ b, int D) {
  float acc = 0.f;
  for (int f0 = 0; f0 < D; f0 += CHUNK) {
    int fl = min(CHUNK, D - f0);
    Kahan k;
    if (METRIC == 1) for (int f = 0; f < fl; f++) k.mac(a[f0 + f], b[f0 + f]);
    else for (int f = 0; f < fl; f++) k.sqdiff(a[f0 + f], b[f0 + f]);
    acc += k.sum;
  }
  return finalize_distance<METRIC>(acc);
}

template <int METRIC>
__global__ void knn_radii_kernel(const float* __restrict__ X, const float* __restrict__ C, uint32_t n,
                                 int D, uint32_t K, const uint32_t* __restrict__ assign,
                                 uint32_t* __restrict__ radii_bits) {
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  uint32_t a = assign[i];
  if (a >= K) return;
  float d = chunked_distance<METRIC, 16>(X + static_cast<size_t>(i) * D, C + static_cast<size_t>(a) * D, D);
  if (d == d) atomicMax(radii_bits + a, __float_as_uint(fmaxf(d, 0.f)));
}

__global__ void knn_radii_fix_kernel(const uint32_t* __restrict__ assign_counts_off, uint32_t K,
                                     float* __restrict__ radii) {
  uint32_t c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= K) return;
  if (assign_counts_off[c + 1] == assign_counts_off[c]) radii[c] = __int_as_float(0x7fc00000);
}

cudaError_t launch_knn_radii(int metric, const float* X, const float* C, uint32_t n, int D, uint32_t K,
                             const uint32_t* assign, float* radii, cudaStream_t st) {
  cudaMemsetAsync(radii, 0, sizeof(float) * K, st);
  if (n == 0) return cudaGetLastError();
  if (metric == 1)
    knn_radii_kernel<1><<<cdiv(n, 256), 256, 0, st>>>(X, C, n, D, K, assign, reinterpret_cast<uint32_t*>(radii));
  else
    knn_radii_kernel<0><<<cdiv(n, 256), 256, 0, st>>>(X, C, n, D, K, assign, reinterpret_cast<uint32_t*>(radii));
  return cudaGetLastError();
}

template <int METRIC>
__global__ void knn_cdist_kernel(const float* __restrict__ C, uint32_t K, int D, float* __restrict__ cd) {
  size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= static_cast<size_t>(K) * K) return;
  uint32_t a = i / K, b = i - static_cast<size_t>(a) * K;
  // the reference fills the upper triangle and mirrors it (knn.cu:60-131): evaluate (min,max) order
  uint32_t lo = min(a, b), hi = max(a, b);
  cd[i] = chunked_distance<METRIC, 24>(C + static_cast<size_t>(lo) * D, C + static_cast<size_t>(hi) * D, D);
}

cudaError_t launch_knn_centroid_distances(int metric, const float* C, uint32_t K, int D, float* cd,
                                          cudaStream_t st) {
  size_t n = static_cast<size_t>(K) * K;
  if (metric == 1) knn_cdist_kernel<1><<<cdiv(n, 128), 128, 0, st>>>(C, K, D, cd);
  else knn_cdist_kernel<0><<<cdiv(n, 128), 128, 0, st>>>(C, K, D, cd);
  return cudaGetLastError();
}

// ------------------------------------------------------------------------------------------------
// Exact cluster-pruned search for the queries the tensor-core pass does not serve (angular metric, k > 15,
// D % 4 != 0 or D > 512, tiny inputs, rows with non-finite data).  One WARP per query:
//   * the query row sits in shared memory, the 32 lanes evaluate 32 candidates of a cluster at a time (every lane
//     streams its own candidate row; the exact distance is the reference's Kahan / round-down-FMA sequence of
//     exact.cuh, so the decisions are the reference's);
//   * the k best so far are a SORTED list (distance ascending) in the query's scratch slice, maintained by the whole
//     warp: position by ballot + popcount, shift by one, insert -- no per-thread heap, and the output is the list
//     itself;
//   * clusters are visited and skipped by the reference's rule `Cd[B][A] - d(q, A) - R[B] > kth` (knn.cu:218-225),
//     candidates enter on `dist <= kth` (knn.cu:204,234); a candidate equal to the current k-th distance displaces
//     it, as a heap replacement does.
// ------------------------------------------------------------------------------------------------
constexpr int kKnnWarps = 8;           // queries per CTA
constexpr int kKnnMaxSmemD = 2048;     // features of the query row kept in shared memory (else read through L1)

// insert (d, o) into the ascending list ld[0..k) / li[0..k) of this warp's query; returns the new k-th distance
__device__ __forceinline__ float knn_list_insert(int k, int lane, float d, uint32_t o, float* ld, uint32_t* li) {
  // position = number of entries strictly smaller than d (the new element goes in front of its equals)
  int pos = 0;
  for (int j0 = 0; j0 < k; j0 += 32) {
    const int j = j0 + lane;
    const bool less = j < k && ld[j] < d;
    pos += __popc(__ballot_sync(0xffffffffu, less));
  }
  // shift [pos, k-2] one place up, highest chunk first so that no entry is overwritten before it is read
  for (int j0 = ((k - 1) / 32) * 32; j0 >= 0; j0 -= 32) {
    const int j = j0 + lane;
    float vd = 0.f;
    uint32_t vi = 0;
    const bool mv = j >= pos && j < k - 1;
    if (mv) { vd = ld[j]; vi = li[j]; }
    __syncwarp();
    if (mv) { ld[j + 1] = vd; li[j + 1] = vi; }
    __syncwarp();
  }
  if (lane == 0) { ld[pos] = d; li[pos] = o; }
  __syncwarp();
  return ld[k - 1];
}

template <int METRIC>
__global__ void __launch_bounds__(kKnnWarps * 32)
knn_warp_search_kernel(int k, const float* __restrict__ X, const float* __restrict__ C, uint32_t N, int D,
                       uint32_t K, uint32_t q_offset, uint32_t q_length, const uint32_t* __restrict__ assign,
                       const uint32_t* __restrict__ inv, const uint32_t* __restrict__ inv_off,
                       const float* __restrict__ cd, const float* __restrict__ radii,
                       float* __restrict__ scratch, uint32_t* __restrict__ neighbors,
                       unsigned long long* __restrict__ d_pairs,
                       // list mode (rows != nullptr): the queries are rows[0 .. *d_nrows), scratch slice = list slot
                       const uint32_t* __restrict__ rows, const uint32_t* __restrict__ d_nrows, int smem_d) {
  extern __shared__ float s_query[];   // [kKnnWarps][smem_d]
  const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
  const uint32_t count = rows ? min(*d_nrows, q_length) : q_length;
  const uint32_t nwarps = gridDim.x * kKnnWarps;
  for (uint32_t q = blockIdx.x * kKnnWarps + wib; q < count; q += nwarps) {
    const uint32_t s = rows ? rows[q] : q_offset + q;
    const uint32_t oq = s - q_offset;          // output row
    const float* xg = X + static_cast<size_t>(s) * D;
    const float* xs = xg;
    if (smem_d) {
      float* mine = s_query + static_cast<size_t>(wib) * smem_d;
      __syncwarp();
      for (int f = lane; f < D; f += 32) mine[f] = xg[f];
      __syncwarp();
      xs = mine;
    }
    float* ld = scratch + static_cast<size_t>(q) * 2 * k;
    uint32_t* li = reinterpret_cast<uint32_t*>(ld + k);
    for (int j = lane; j < k; j += 32) { ld[j] = FLT_MAX; li[j] = UINT32_MAX; }
    __syncwarp();
    const uint32_t A = assign[s];
    unsigned long long pairs = 0;
    float kth = FLT_MAX;
    float dA = 0.f;
    if (A < K) dA = distance_exact<METRIC>(xs, C + static_cast<size_t>(A) * D, D);   // every lane: same value
    // own cluster first, then the others in ascending order; B == K + 1 ends the walk
    for (uint32_t step = 0; step <= K; step++) {
      uint32_t B;
      if (step == 0) {
        if (A >= K) continue;
        B = A;
      } else {
        B = step - 1;
        if (B == A) continue;
        const float cdist = A < K ? cd[static_cast<size_t>(B) * K + A] : 0.f;
        if (cdist != cdist) continue;
        if (A < K && cdist - dA - radii[B] > kth) continue;
      }
      const uint32_t b = inv_off[B], e = inv_off[B + 1];
      pairs += e - b;
      for (uint32_t p0 = b; p0 < e; p0 += 32) {
        const uint32_t pp = p0 + lane;
        uint32_t o = UINT32_MAX;
        float d = FLT_MAX;
        bool want = false;
        if (pp < e) {
          o = inv[pp];
          if (o != s) {
            d = distance_exact<METRIC>(xs, X + static_cast<size_t>(o) * D, D);
            want = d <= kth;
          }
        }
        unsigned m = __ballot_sync(0xffffffffu, want);
        while (m) {                          // arrival order = position order, as in the reference's sequential scan
          const int src = __ffs(m) - 1;
          m &= m - 1;
          const float dd = __shfl_sync(0xffffffffu, d, src);
          const uint32_t oo = __shfl_sync(0xffffffffu, o, src);
          if (dd <= kth) kth = knn_list_insert(k, lane, dd, oo, ld, li);
        }
      }
    }
    __syncwarp();
    for (int j = lane; j < k; j += 32) neighbors[static_cast<size_t>(oq) * k + j] = li[j];
    if (lane == 0) atomicAdd(d_pairs, pairs);
  }
}

cudaError_t launch_knn_search(int metric, int k, const float* X, const float* C, uint32_t N, int D,
                              uint32_t K, uint32_t q_offset, uint32_t q_length, const uint32_t* assign,
                              const uint32_t* inv, const uint32_t* inv_off, const float* cd,
                              const float* radii, float* heap_scratch, uint32_t* neighbors,
                              unsigned long long* d_pairs, const uint32_t* rows, const uint32_t* d_nrows,
                              cudaStream_t st) {
  if (q_length == 0) return cudaSuccess;
  const int smem_d = D <= kKnnMaxSmemD ? D : 0;
  const size_t smem = static_cast<size_t>(kKnnWarps) * smem_d * sizeof(float);
  const unsigned grid = rows ? device_sms() * 8u : static_cast<unsigned>(std::min<size_t>(cdiv(q_length, kKnnWarps), device_sms() * 64u));
  cudaError_t e;
  if (metric == 1) {
    if ((e = cudaFuncSetAttribute(knn_warp_search_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                  static_cast<int>(smem))) != cudaSuccess) return e;
    knn_warp_search_kernel<1><<<grid, kKnnWarps * 32, smem, st>>>(k, X, C, N, D, K, q_offset, q_length, assign, inv, inv_off,
                                                                  cd, radii, heap_scratch, neighbors, d_pairs, rows, d_nrows,
                                                                  smem_d);
  } else {
    if ((e = cudaFuncSetAttribute(knn_warp_search_kernel<0>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                  static_cast<int>(smem))) != cudaSuccess) return e;
    knn_warp_search_kernel<0><<<grid, kKnnWarps * 32, smem, st>>>(k, X, C, N, D, K, q_offset, q_length, assign, inv, inv_off,
                                                                  cd, radii, heap_scratch, neighbors, d_pairs, rows, d_nrows,
                                                                  smem_d);
  }
  return cudaGetLastError();
}

// empty clusters have no radius (NaN, knn.cu:56); run once after launch_knn_radii + the inverse assignment
cudaError_t launch_knn_radii_fix(const uint32_t* inv_off, uint32_t K, float* radii, cudaStream_t st) {
  knn_radii_fix_kernel<<<cdiv(K, 128), 128, 0, st>>>(inv_off, K, radii);
  return cudaGetLastError();
}

// rows of the sorted order past `nv` (samples whose assignment is not a valid cluster) join the exact-search list
__global__ void knn_tail_rows_kernel(const uint32_t* __restrict__ inv, uint32_t nv, uint32_t n,
                                     uint32_t* __restrict__ rows, uint32_t* __restrict__ d_nrows) {
  uint32_t i = nv + blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) rows[atomicAdd(d_nrows, 1u)] = inv[i];
}
cudaError_t launch_knn_tail_rows(const uint32_t* inv, uint32_t nv, uint32_t n, uint32_t* rows, uint32_t* d_nrows,
                                 cudaStream_t st) {
  if (nv >= n) return cudaSuccess;
  knn_tail_rows_kernel<<<cdiv(n - nv, 256), 256, 0, st>>>(inv, nv, n, rows, d_nrows);
  return cudaGetLastError();
}

}  // namespace kmb
