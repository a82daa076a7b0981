// exact.cuh -- the reference's fp32 distance arithmetic, restated for the exact ("re-check") kernels.
//
// The tensor-core kernel (assign_tc.cu) only *filters*: every assignment / neighbour decision that
// leaves this library is made by the functions below, which reproduce the instruction sequence of
// the reference bit for bit (SURVEY.md Appendix A):
//
//   fma_rd(a,b,c)      = __fmaf_rd(a,b,c)                     reference fp_abstraction.h:88-90
//   Kahan "inverted c" = y=fma_rd(a,b,r); t=p+y; r=y-(t-p)    reference kmeans.cu:331-341
//   L2 ranking score   = fma_rd(-2, dot, 0+csqr)              reference metric_abstraction.h:55-57
//   cos ranking score  = clamp-acosf(dot)                     reference metric_abstraction.h:171-177
//   true distances     = sqrt_rn(Kahan sum (a-b)^2) / acosf   reference metric_abstraction.h:59-101,179-222
//
// No fast-math: none of these bodies contains a contractible mul+add pair besides the explicit
// intrinsics, so nvcc's default -fmad=true cannot change them.
#pragma once
#include <cuda_runtime.h>
#include <cfloat>
#include <cstdint>

namespace kmb {

#ifndef M_PI_F
#define M_PI_F 3.14159265358979323846f
#endif

struct Kahan {
  float sum, corr;
  __device__ __forceinline__ Kahan() : sum(0.f), corr(0.f) {}
  // one step of sum += a*b
  __device__ __forceinline__ void mac(float a, float b) {
    float y = __fmaf_rd(a, b, corr);
    float t = sum + y;
    corr = y - (t - sum);
    sum = t;
  }
  // one step of sum += (a-b)^2
  __device__ __forceinline__ void sqdiff(float a, float b) {
    float d = a - b;
    mac(d, d);
  }
};

__device__ __forceinline__ float acos_clamped(float p) {
  if (p >= 1.f) return 0.f;
  if (p <= -1.f) return M_PI_F;
  return acosf(p);
}

template <int METRIC>  // 0 = L2, 1 = cosine
__device__ __forceinline__ float lloyd_score(float dot, float csqr) {
  if (METRIC == 1) return acos_clamped(dot);
  return __fmaf_rd(-2.f, dot, 0.f + csqr);
}

template <int METRIC>
__device__ __forceinline__ float finalize_distance(float partial) {
  if (METRIC == 1) return acos_clamped(partial);
  return __fsqrt_rn(partial);
}

// ||c||^2 as the reference computes it (constant 1 for cosine): metric_abstraction.h:21-36,149-158
template <int METRIC>
__device__ __forceinline__ float csqr_exact(const float* __restrict__ c, int D) {
  if (METRIC == 1) return 1.f;
  Kahan k;
  for (int f = 0; f < D; f++) {
    float v = c[f];
    k.mac(v, v);
  }
  return k.sum;
}

// true distance between two row-major vectors in global/shared memory
template <int METRIC>
__device__ __forceinline__ float distance_exact(const float* __restrict__ a,
                                                const float* __restrict__ b, int D) {
  Kahan k;
  if (METRIC == 1) {
    for (int f = 0; f < D; f++) k.mac(a[f], b[f]);
  } else {
    for (int f = 0; f < D; f++) k.sqdiff(a[f], b[f]);
  }
  return finalize_distance<METRIC>(k.sum);
}

// The staged pass of the per-row kernels (k-means|| update, greedy k-means++ trials, mini-batch inertia, relocation
// keys, restart inertia): kStagedRows rows per CTA, one thread per row, 32-feature slices of the rows staged through
// padded shared memory (coalesced loads), then every thread advances the sequential Kahan chain of its own row.
constexpr int kStagedRows = 128;

// the sample rows row0, row0 + 1, ... of a CTA, indexed as s_row[] is
struct RowRange {
  uint32_t row0;
  __device__ __forceinline__ uint32_t operator[](int r) const { return row0 + r; }
};

// tile[r * 33 + f] = feature f0 + f of sample rows[r] for the fl features of the slice, 0 past them and on the padding
// rows (row0 + r >= n); rows is s_row[] (shared memory) or a RowRange; tile holds kStagedRows * 33 floats
template <class Rows>
__device__ __forceinline__ void stage_slice(const float* __restrict__ X, const Rows& rows, uint32_t row0, uint32_t n,
                                            int D, int f0, int fl, float* tile) {
  const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
#pragma unroll 8
  for (int rr = 0; rr < 32; rr++) {   // warp w stages rows w, w + 4, ...: one coalesced 128-byte segment per row
    const int r = warp + 4 * rr;
    tile[r * 33 + lane] = (row0 + r < n && lane < fl) ? X[static_cast<size_t>(rows[r]) * D + f0 + lane] : 0.f;
  }
}

// The staged pass against each row's own centroid `c`, read as float4 when VEC4 (D % 4 == 0).  Returns the Kahan sum
// of (x - c)^2 (METRIC 0) or of x * c (METRIC 1) in the reference's order; meaningful only where `live`.
template <bool VEC4, int METRIC, class Rows>
__device__ __forceinline__ float staged_own_sum(const float* __restrict__ X, const Rows& rows, uint32_t row0,
                                                uint32_t n, int D, const float* __restrict__ c, bool live,
                                                float* tile) {
  const int t = threadIdx.x;
  Kahan k;
  for (int f0 = 0; f0 < D; f0 += 32) {
    const int fl = min(32, D - f0);
    stage_slice(X, rows, row0, n, D, f0, fl, tile);
    __syncthreads();
    if (live) {
      const float* xs = tile + t * 33;
      if (VEC4 && fl == 32) {
#pragma unroll
        for (int q = 0; q < 8; q++) {
          const float4 cv = __ldg(reinterpret_cast<const float4*>(c + f0) + q);
          if (METRIC == 1) {
            k.mac(xs[4 * q], cv.x); k.mac(xs[4 * q + 1], cv.y);
            k.mac(xs[4 * q + 2], cv.z); k.mac(xs[4 * q + 3], cv.w);
          } else {
            k.sqdiff(xs[4 * q], cv.x); k.sqdiff(xs[4 * q + 1], cv.y);
            k.sqdiff(xs[4 * q + 2], cv.z); k.sqdiff(xs[4 * q + 3], cv.w);
          }
        }
      } else {
        for (int f = 0; f < fl; f++) {
          if (METRIC == 1) k.mac(xs[f], __ldg(c + f0 + f));
          else k.sqdiff(xs[f], __ldg(c + f0 + f));
        }
      }
    }
    __syncthreads();
  }
  return k.sum;
}

}  // namespace kmb
