// fixed_order.cuh -- the deterministic building blocks of the seeding, mini-batch, relocation and restart kernels.
//
// The draws are stateless counter hashes of the global row index, so they are the same on any number of GPUs and for
// any launch shape; the double totals are added in an order that depends only on the number of terms (no atomics).
// Every kernel that makes one of these promises uses the functions below, so the promises cannot drift apart.
#pragma once
#include <cuda_runtime.h>
#include <cstdint>

namespace kmb {

// SplitMix64's finaliser
__host__ __device__ __forceinline__ uint64_t splitmix64(uint64_t z) {
  z += 0x9E3779B97F4A7C15ull;
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  return z ^ (z >> 31);
}

// the top 53 bits of a hash as a double in [0, 1)
__device__ __forceinline__ double unit_co(uint64_t h) { return static_cast<double>(h >> 11) * (1.0 / 9007199254740992.0); }

// the top 53 bits of a hash as a double in (0, 1), for -log(u)
__device__ __forceinline__ double unit_oo(uint64_t h) {
  return (static_cast<double>(h >> 11) + 0.5) * (1.0 / 9007199254740992.0);
}

// the d^2 draws' mass w d^2 in double; rows with a non-finite distance carry none
__device__ __forceinline__ double d2_mass(float d, float w) {
  if (!isfinite(d)) return 0.0;
  const double dd = static_cast<double>(d);
  return static_cast<double>(w) * (dd * dd);
}

// The CTA's sum of v, returned on thread 0: a shuffle tree per warp, then thread 0 adds the warps in order starting
// from 0.0.  s_part holds THREADS / 32 doubles; another call may reuse it after a __syncthreads().
template <int THREADS>
__device__ __forceinline__ double block_sum(double v, double* s_part) {
  const int t = threadIdx.x;
  for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
  if ((t & 31) == 0) s_part[t >> 5] = v;
  __syncthreads();
  double s = 0.0;
  if (t == 0)
    for (int q = 0; q < THREADS / 32; q++) s += s_part[q];
  return s;
}

// The fixed-order total of n doubles by one 1024-thread CTA, in two steps: thread t adds its contiguous chunk
// [lo, hi) of ceil(n / 1024) terms in index order (chunk_sum), then one thread adds the 1024 chunk sums in order
// (fold_chunks).
__device__ __forceinline__ void chunk_range(uint32_t n, uint32_t& lo, uint32_t& hi) {
  const uint32_t per = (n + 1023) / 1024;
  lo = min(n, threadIdx.x * per);
  hi = min(n, lo + per);
}

// FINITE_ONLY: a term that is not finite adds 0 (the centre-shift total, where a dead centroid's NaN must not count)
template <bool FINITE_ONLY = false>
__device__ __forceinline__ double chunk_sum(const double* __restrict__ v, uint32_t n) {
  uint32_t lo, hi;
  chunk_range(n, lo, hi);
  double acc = 0.0;
  for (uint32_t b = lo; b < hi; b++) {
    if constexpr (FINITE_ONLY) acc += isfinite(v[b]) ? v[b] : 0.0;
    else acc += v[b];
  }
  return acc;
}

__device__ __forceinline__ double fold_chunks(const double* s_chunk) {
  double s = 0.0;
  for (int q = 0; q < 1024; q++) s += s_chunk[q];
  return s;
}

}  // namespace kmb
