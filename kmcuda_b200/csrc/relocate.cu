// relocate.cu -- device side of the empty-cluster relocation of the Lloyd / Yinyang update (relocate_empty_clusters,
// DESIGN.md §4l; the host walk is Job::relocate in job.cu).  When a cluster has no members after the exchange, it takes
// one of the rows farthest from their own centroid, as scikit-learn's _relocate_empty_clusters_dense does:
//   keys     one staged pass over the shard (staged_own_sum, the mini-batch inertia body): key_i = the orderable bits
//            of d_i in the high word, ~global row in the low word, so one descending order is (d desc, row asc);
//            0 for a row that is not eligible (no centroid, weight 0, d not finite)
//   select   the top T keys without sorting all of them: 8-bit radix-select passes over the keys find a threshold
//            that at most cap keys reach, cub::DeviceSelect takes those, cub::DeviceRadixSort orders them
//   apply    in walk order: sums[donor] -= w x, counts[donor] -= 1, W[donor] -= w; sums[e] = w x, counts[e] = 1,
//            W[e] = w; after the normalisation the angular centroid of e is overwritten with x / ||x||
// The restarts' inertia pass (Job::restarts, DESIGN.md §4n) sums w e over the rows the keys pass would find eligible,
// with the same staged row distance.
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_select.cuh>

#include <algorithm>

#include "exact.cuh"
#include "fixed_order.cuh"
#include "shard.h"

namespace kmb {

namespace {

// The rule both the relocation keys and the inertia apply to shard row i of the CTA (kStagedRows threads): eligible
// when assign[i] < K, w_i > 0 (w optional) and its distance d to its own centroid is finite; d = the L2 Kahan sum of
// squared differences (before the square root) or the angle (METRIC 1).  wi = w_i (0 past the shard), d is set only
// where eligible.
template <bool VEC4, int METRIC>
__device__ __forceinline__ bool eligible_own_distance(const float* __restrict__ X, uint32_t n, int D,
                                                      const float* __restrict__ C, uint32_t K,
                                                      const uint32_t* __restrict__ assign, const float* __restrict__ w,
                                                      uint32_t* s_row, float* tile, float& d, float& wi) {
  const int t = threadIdx.x;
  const uint32_t row0 = blockIdx.x * kStagedRows, i = row0 + t;
  uint32_t a = K;
  wi = 0.f;
  if (i < n) {
    a = min(assign[i], K);
    wi = w ? w[i] : 1.f;
  }
  const bool live = a < K && wi > 0.f;
  const float* c = C + static_cast<size_t>(live ? a : 0) * D;
  s_row[t] = i < n ? i : 0u;
  __syncthreads();
  const float sum = staged_own_sum<VEC4, METRIC>(X, s_row, row0, n, D, c, live, tile);
  if (!live) return false;
  d = METRIC == 1 ? acos_clamped(sum) : sum;
  return isfinite(d);
}

template <bool VEC4, int METRIC>
__global__ void __launch_bounds__(kStagedRows)
reloc_keys_kernel(const float* __restrict__ X, uint32_t n, int D, const float* __restrict__ C, uint32_t K,
                  const uint32_t* __restrict__ assign, const float* __restrict__ w, uint32_t off,
                  uint64_t* __restrict__ keys) {
  __shared__ uint32_t s_row[kStagedRows];
  __shared__ float tile[kStagedRows * 33];
  const uint32_t i = blockIdx.x * kStagedRows + threadIdx.x;
  float d, wi;
  const bool eligible = eligible_own_distance<VEC4, METRIC>(X, n, D, C, K, assign, w, s_row, tile, d, wi);
  if (i < n) {
    uint64_t key = 0;
    if (eligible) {
      const uint32_t b = __float_as_uint(d);
      const uint32_t ob = (b & 0x80000000u) ? ~b : (b | 0x80000000u);
      key = (static_cast<uint64_t>(ob) << 32) | static_cast<uint32_t>(~(off + i));
    }
    keys[i] = key;
  }
}

// Inertia of a run (restarts, DESIGN.md §4n): sum of w e over the block's eligible rows, e = d (L2: the Kahan sum of
// squared differences) or d^2 (angular: the angle), into bsum[block] (block_sum).
template <bool VEC4, int METRIC>
__global__ void __launch_bounds__(kStagedRows)
inertia_kernel(const float* __restrict__ X, uint32_t n, int D, const float* __restrict__ C, uint32_t K,
               const uint32_t* __restrict__ assign, const float* __restrict__ w, double* __restrict__ bsum) {
  __shared__ uint32_t s_row[kStagedRows];
  __shared__ float tile[kStagedRows * 33];
  __shared__ double s_part[kStagedRows / 32];
  float d, wi;
  double m = 0.0;
  if (eligible_own_distance<VEC4, METRIC>(X, n, D, C, K, assign, w, s_row, tile, d, wi))
    m = static_cast<double>(wi) * (METRIC == 1 ? static_cast<double>(d) * d : static_cast<double>(d));
  const double s = block_sum<kStagedRows>(m, s_part);
  if (threadIdx.x == 0) bsum[blockIdx.x] = s;
}

// one radix-select pass: histogram of the 8-bit digit at `shift` over the eligible keys whose higher digits equal the
// prefix found so far
__global__ void __launch_bounds__(256)
reloc_hist_kernel(const uint64_t* __restrict__ keys, uint32_t n, int shift, const RelocState* s,
                  uint32_t* __restrict__ hist) {
  if (s->done) return;
  __shared__ uint32_t h[256];
  h[threadIdx.x] = 0;
  __syncthreads();
  const uint64_t prefix = s->prefix;
  const size_t stride = static_cast<size_t>(gridDim.x) * blockDim.x;
  for (size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += stride) {
    const uint64_t k = keys[i];
    if (k && (shift == 56 || (k >> (shift + 8)) == prefix)) atomicAdd(&h[(k >> shift) & 255u], 1u);
  }
  __syncthreads();
  if (h[threadIdx.x]) atomicAdd(&hist[threadIdx.x], h[threadIdx.x]);
}

// the digit of the T-th largest key; done once at most cap keys reach the threshold (or every digit is fixed)
__global__ void reloc_scan_kernel(uint32_t* __restrict__ hist, int shift, uint32_t T, uint32_t cap, RelocState* s) {
  if (s->done) return;
  bool done = false;
  if (shift == 56) {
    uint32_t e = 0;
    for (int b = 0; b < 256; b++) e += hist[b];
    s->eligible = e;
    if (e <= T) {
      s->thr = 1;
      done = true;
    }
  }
  if (!done) {
    uint32_t cum = s->above;
    int d = 255;
    for (; d > 0; d--) {
      if (cum + hist[d] >= T) break;
      cum += hist[d];
    }
    s->prefix = (s->prefix << 8) | static_cast<uint64_t>(d);
    s->above = cum;
    if (cum + hist[d] <= cap || shift == 0) {
      s->thr = max(s->prefix << shift, static_cast<uint64_t>(1));   // key 0 is never selected
      done = true;
    }
  }
  s->done = done ? 1u : 0u;
  for (int b = 0; b < 256; b++) hist[b] = 0;
}

struct AtLeast {
  const uint64_t* thr;
  __device__ __forceinline__ bool operator()(uint64_t k) const { return k >= *thr; }
};

// donor and weight of each listed key (rows of this shard, global index ~low word)
__global__ void reloc_gather_kernel(const uint64_t* __restrict__ top, uint32_t T, uint32_t off,
                                    const uint32_t* __restrict__ assign, const float* __restrict__ w,
                                    uint32_t* __restrict__ meta) {
  const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= T) return;
  const uint64_t k = top[j];
  uint32_t donor = 0xFFFFFFFFu;
  float wj = 0.f;
  if (k) {
    const uint32_t i = ~static_cast<uint32_t>(k) - off;
    donor = assign[i];
    wj = w ? w[i] : 1.f;
  }
  meta[2 * j] = donor;
  meta[2 * j + 1] = __float_as_uint(wj);
}

// one thread per feature walks the relocations in order (several picks from one donor subtract in walk order); the
// first thread also moves the counts and weight totals.  meta: [3r] = cluster, donor, weight bits
__global__ void reloc_apply_kernel(float* __restrict__ sums, uint32_t* __restrict__ counts, float* __restrict__ wsums,
                                   int D, const float* __restrict__ xs, const uint32_t* __restrict__ meta, uint32_t r) {
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f < D) {
    for (uint32_t j = 0; j < r; j++) {
      const uint32_t e = meta[3 * j], a = meta[3 * j + 1];
      const float wx = __fmul_rn(__uint_as_float(meta[3 * j + 2]), xs[static_cast<size_t>(j) * D + f]);
      float* sa = sums + static_cast<size_t>(a) * D + f;
      *sa = __fsub_rn(*sa, wx);
      sums[static_cast<size_t>(e) * D + f] = wx;
    }
  }
  if (f == 0) {
    for (uint32_t j = 0; j < r; j++) {
      const uint32_t e = meta[3 * j], a = meta[3 * j + 1];
      const float wj = __uint_as_float(meta[3 * j + 2]);
      counts[a] -= 1;
      counts[e] = 1;
      if (wsums) {
        wsums[a] = __fsub_rn(wsums[a], wj);
        wsums[e] = wj;
      }
    }
  }
}

// angular: the relocated centroid is x normalised in the reference's order (normalize_kernel<1>)
__global__ void reloc_cos_overwrite_kernel(float* __restrict__ C, int D, const float* __restrict__ xs,
                                           const uint32_t* __restrict__ meta, uint32_t r) {
  const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= r) return;
  const float* x = xs + static_cast<size_t>(j) * D;
  float* o = C + static_cast<size_t>(meta[3 * j]) * D;
  Kahan k;
  for (int f = 0; f < D; f++) k.mac(x[f], x[f]);
  const float scale = __frcp_rn(__fsqrt_rn(k.sum));
  for (int f = 0; f < D; f++) o[f] = x[f] * scale;
}

}  // namespace

cudaError_t launch_reloc_keys(int metric, const float* X, uint32_t n, int D, const float* C, uint32_t K,
                              const uint32_t* assign, const float* w, uint32_t off, uint64_t* keys, cudaStream_t st) {
  if (n == 0) return cudaSuccess;
  const unsigned grid = cdiv(n, kStagedRows);
  const bool v4 = D % 4 == 0;
  if (metric == 1) {
    if (v4) reloc_keys_kernel<true, 1><<<grid, kStagedRows, 0, st>>>(X, n, D, C, K, assign, w, off, keys);
    else reloc_keys_kernel<false, 1><<<grid, kStagedRows, 0, st>>>(X, n, D, C, K, assign, w, off, keys);
  } else {
    if (v4) reloc_keys_kernel<true, 0><<<grid, kStagedRows, 0, st>>>(X, n, D, C, K, assign, w, off, keys);
    else reloc_keys_kernel<false, 0><<<grid, kStagedRows, 0, st>>>(X, n, D, C, K, assign, w, off, keys);
  }
  return cudaGetLastError();
}

uint32_t inertia_blocks(uint32_t n) { return std::max(1u, cdiv(n, kStagedRows)); }

cudaError_t launch_inertia(int metric, const float* X, uint32_t n, int D, const float* C, uint32_t K,
                           const uint32_t* assign, const float* w, double* bsum, double* out, cudaStream_t st) {
  if (n == 0) return cudaMemsetAsync(out, 0, sizeof(double), st);
  const unsigned grid = cdiv(n, kStagedRows);
  const bool v4 = D % 4 == 0;
  if (metric == 1) {
    if (v4) inertia_kernel<true, 1><<<grid, kStagedRows, 0, st>>>(X, n, D, C, K, assign, w, bsum);
    else inertia_kernel<false, 1><<<grid, kStagedRows, 0, st>>>(X, n, D, C, K, assign, w, bsum);
  } else {
    if (v4) inertia_kernel<true, 0><<<grid, kStagedRows, 0, st>>>(X, n, D, C, K, assign, w, bsum);
    else inertia_kernel<false, 0><<<grid, kStagedRows, 0, st>>>(X, n, D, C, K, assign, w, bsum);
  }
  cudaError_t e = cudaGetLastError();
  return e == cudaSuccess ? launch_fixed_sum(bsum, grid, out, st) : e;
}

uint32_t reloc_cap(uint32_t T) { return 2 * T + 4096; }

size_t reloc_select_bytes(uint32_t n, uint32_t cap) {
  size_t b1 = 0, b2 = 0;
  cub::DeviceSelect::If(nullptr, b1, static_cast<const uint64_t*>(nullptr), static_cast<uint64_t*>(nullptr),
                        static_cast<uint32_t*>(nullptr), static_cast<int>(std::max(n, 1u)), AtLeast{nullptr});
  cub::DeviceRadixSort::SortKeysDescending(nullptr, b2, static_cast<const uint64_t*>(nullptr),
                                           static_cast<uint64_t*>(nullptr), static_cast<int>(cap));
  return std::max(b1, b2);
}

cudaError_t launch_reloc_select(const RelocSelect& s, cudaStream_t st) {
  cudaError_t e;
  if ((e = cudaMemsetAsync(s.state, 0, sizeof(RelocState), st)) != cudaSuccess) return e;
  if ((e = cudaMemsetAsync(s.hist, 0, sizeof(uint32_t) * 256, st)) != cudaSuccess) return e;
  if ((e = cudaMemsetAsync(s.sel, 0, sizeof(uint64_t) * s.cap, st)) != cudaSuccess) return e;
  const unsigned grid = static_cast<unsigned>(std::min<size_t>(device_sms() * 4, cdiv(std::max(s.n, 1u), 256)));
  for (int shift = 56; shift >= 0; shift -= 8) {
    reloc_hist_kernel<<<grid, 256, 0, st>>>(s.keys, s.n, shift, s.state, s.hist);
    reloc_scan_kernel<<<1, 1, 0, st>>>(s.hist, shift, s.T, s.cap, s.state);
  }
  if ((e = cudaGetLastError()) != cudaSuccess) return e;
  size_t bytes = s.tmp_bytes;
  if ((e = cub::DeviceSelect::If(s.tmp, bytes, s.keys, s.sel, s.nsel, static_cast<int>(s.n), AtLeast{&s.state->thr},
                                 st)) != cudaSuccess)
    return e;
  bytes = s.tmp_bytes;
  return cub::DeviceRadixSort::SortKeysDescending(s.tmp, bytes, s.sel, s.top, static_cast<int>(s.cap), 0, 64, st);
}

cudaError_t launch_reloc_gather(const uint64_t* top, uint32_t T, uint32_t off, const uint32_t* assign, const float* w,
                                uint32_t* meta, cudaStream_t st) {
  if (T == 0) return cudaSuccess;
  reloc_gather_kernel<<<cdiv(T, 256), 256, 0, st>>>(top, T, off, assign, w, meta);
  return cudaGetLastError();
}

cudaError_t launch_reloc_apply(float* sums, uint32_t* counts, float* wsums, int D, const float* xs,
                               const uint32_t* meta, uint32_t r, cudaStream_t st) {
  if (r == 0) return cudaSuccess;
  reloc_apply_kernel<<<cdiv(D, 128), 128, 0, st>>>(sums, counts, wsums, D, xs, meta, r);
  return cudaGetLastError();
}

cudaError_t launch_reloc_cos_overwrite(float* C, int D, const float* xs, const uint32_t* meta, uint32_t r,
                                       cudaStream_t st) {
  if (r == 0) return cudaSuccess;
  reloc_cos_overwrite_kernel<<<cdiv(r, 64), 64, 0, st>>>(C, D, xs, meta, r);
  return cudaGetLastError();
}

}  // namespace kmb

extern "C" {

// ---- diagnostics (used by tests; not part of the drop-in surface) ----
// The relocation keys of samples [n][D] against centroids [K][D] and assignments [n] (weights [n] or NULL), global row
// = local row, into keys_out [n], and the T largest (descending, 0 = no more eligible rows) into top_out [T].  Device
// pointers on the current device, default stream, synchronous.  Returns the number of eligible rows, or -1.
int64_t kmcuda_b200_debug_relocate_select(int32_t metric, uint32_t n, uint16_t features_size, const float* samples,
                                          const float* centroids, uint32_t clusters_size, const uint32_t* assignments,
                                          const float* weights, uint32_t T, uint64_t* keys_out, uint64_t* top_out) {
  using namespace kmb;
  if (!samples || !centroids || !assignments || !keys_out || !top_out || T == 0 || n == 0) return -1;
  const uint32_t cap = reloc_cap(T);
  DevBuf<uint64_t> state, sel, top;
  DevBuf<uint32_t> hist, nsel;
  DevBuf<char> tmp;
  RelocSelect s;
  s.n = n;
  s.T = T;
  s.cap = cap;
  s.keys = keys_out;
  s.tmp_bytes = reloc_select_bytes(n, cap);
  if (state.alloc(sizeof(RelocState) / sizeof(uint64_t)) != cudaSuccess || sel.alloc(cap) != cudaSuccess ||
      top.alloc(cap) != cudaSuccess || hist.alloc(256) != cudaSuccess || nsel.alloc(1) != cudaSuccess ||
      tmp.alloc(s.tmp_bytes) != cudaSuccess)
    return -1;
  s.state = reinterpret_cast<RelocState*>(state.get());
  s.hist = hist;
  s.sel = sel;
  s.top = top;
  s.nsel = nsel;
  s.tmp = tmp.get();
  if (launch_reloc_keys(metric, samples, n, features_size, centroids, clusters_size, assignments, weights, 0, keys_out,
                        nullptr) != cudaSuccess ||
      launch_reloc_select(s, nullptr) != cudaSuccess ||
      cudaMemcpyAsync(top_out, top.get(), sizeof(uint64_t) * T, cudaMemcpyDeviceToDevice, nullptr) != cudaSuccess) {
    cudaDeviceSynchronize();   // the scratch goes back to the pool only once nothing reads it
    return -1;
  }
  RelocState hs;
  if (cudaMemcpy(&hs, s.state, sizeof(hs), cudaMemcpyDeviceToHost) != cudaSuccess) return -1;
  return static_cast<int64_t>(hs.eligible);
}

}  // extern "C"
