// shard.h -- one GPU's share of a clustering job: device buffers + the hot-path steps.
//
// The reference replicates the whole sample matrix on every GPU and splits only the kernel launch
// ranges (kmcuda.cc:139-170, private.h:240-273).  Here a Shard owns just its range of samples and a
// full copy of the (small) centroid table; the caller all-reduces the partial sums between
// partial_sums() and finish_update().
#pragma once
#include <cuda_runtime.h>

#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <utility>
#include <vector>

#include "kernels.h"
#include "kmcuda.h"

namespace kmb {

#define KMB_INFO(...) do { if (verbosity > 0) { printf(__VA_ARGS__); } } while (false)
#define KMB_DEBUG(...) do { if (verbosity > 1) { printf(__VA_ARGS__); } } while (false)

// CUDA call -> KMCUDAResult, logging like the reference's CUCH (private.h:39-48)
#define KMB_CU(call, code)                                                          \
  do {                                                                              \
    cudaError_t kmb_err__ = (call);                                                 \
    if (kmb_err__ != cudaSuccess) {                                                 \
      if (getenv("KMCUDA_B200_DEBUG"))                                              \
        fprintf(stderr, "%s:%d %s -> %s\n", __FILE__, __LINE__, #call, cudaGetErrorString(kmb_err__)); \
      KMB_DEBUG("%s\n", #call);                                                     \
      KMB_INFO("%s:%d -> %s\n", __FILE__, __LINE__, cudaGetErrorString(kmb_err__)); \
      return code;                                                                  \
    }                                                                               \
  } while (false)

#define KMB_RET(call)                            \
  do {                                           \
    KMCUDAResult kmb_res__ = (call);             \
    if (kmb_res__ != kmcudaSuccess) return kmb_res__; \
  } while (false)

// pooled device buffer that frees itself; `borrow` wraps a caller-owned pointer (wrappers.h:16-21)
template <typename T>
class DevBuf {
 public:
  DevBuf() = default;
  DevBuf(const DevBuf&) = delete;
  DevBuf& operator=(const DevBuf&) = delete;
  DevBuf(DevBuf&& o) noexcept : p_(o.p_), owned_(o.owned_) {
    o.p_ = nullptr;
    o.owned_ = false;
  }
  DevBuf& operator=(DevBuf&& o) noexcept {
    if (this != &o) {
      release();
      p_ = o.p_;
      owned_ = o.owned_;
      o.p_ = nullptr;
      o.owned_ = false;
    }
    return *this;
  }
  ~DevBuf() { release(); }
  cudaError_t alloc(size_t n) {
    release();
    if (n == 0) n = 1;
    cudaError_t e = pool_alloc(reinterpret_cast<void**>(&p_), n * sizeof(T));
    owned_ = (e == cudaSuccess);
    if (!owned_) p_ = nullptr;
    return e;
  }
  void borrow(T* p) {
    release();
    p_ = p;
    owned_ = false;
  }
  void release() {
    if (owned_ && p_) pool_free(p_);
    p_ = nullptr;
    owned_ = false;
  }
  T* get() const { return p_; }
  operator T*() const { return p_; }

 private:
  T* p_ = nullptr;
  bool owned_ = false;
};

// equal split of `amount` rows over the devices, chunk starts aligned to 512 bytes (job.cu)
std::vector<std::pair<uint32_t, uint32_t>> split_rows(uint32_t amount, uint32_t row_bytes, size_t ndev);

class Shard {
 public:
  Shard(int metric, int device, uint32_t max_n, int D, uint32_t K, int verbosity)
      : metric(metric), device(device), max_n(max_n), D(D), K(K), verbosity(verbosity) {}
  ~Shard();
  Shard(const Shard&) = delete;

  KMCUDAResult create(bool with_update);
  KMCUDAResult enable_yinyang(uint32_t G);
  KMCUDAResult reset_update_state(cudaStream_t st);
  KMCUDAResult yy_prepare(const uint32_t* host_groups, cudaStream_t st);
  // (re)builds the bounds of every sample of the shard: reference kmeans_yy_init, kmeans.cu:431-485
  KMCUDAResult yy_refresh(uint32_t n, const float* X, const float* C, const uint32_t* assignments, cudaStream_t st);
  KMCUDAResult yy_step(uint32_t n, const float* X, const float* C, uint32_t* assignments, uint32_t* prev,
                       uint32_t* d_changed, cudaStream_t st);

  // hot path
  KMCUDAResult assign(uint32_t n, const float* X, const float* C, uint32_t* assignments,
                      uint32_t* prev, uint32_t* d_changed, cudaStream_t st);
  // mini-batch: result[j] = the winner of sample rows[j] (n <= max_n entries, X has nX rows); row_result [nX] scratch
  KMCUDAResult assign_rows(uint32_t n, const float* X, uint32_t nX, const uint32_t* rows, const float* C,
                           uint32_t* row_result, uint32_t* result, cudaStream_t st);
  // weights (optional, [nX], indexed by row): member sums of the entries rows[0 .. n) with winners keys[0 .. n)
  KMCUDAResult partial_sums_rows(uint32_t n, const float* X, const uint32_t* rows, const uint32_t* keys, float* sums,
                                 uint32_t* counts, cudaStream_t st, const float* weights, float* wsums);
  // weights (optional, [n] on this device): weighted member sums, and wsums[K] = the members' weight totals
  KMCUDAResult partial_sums(uint32_t n, const float* X, const uint32_t* assignments, float* sums,
                            uint32_t* counts, cudaStream_t st, const float* weights = nullptr,
                            float* wsums = nullptr);
  // wsums (optional): normalise by the weight totals; cweights[K] keeps them for the next cosine update
  KMCUDAResult finish_update(const float* sums, const uint32_t* counts, float* C, uint32_t* ccounts,
                             cudaStream_t st, const float* wsums = nullptr, float* cweights = nullptr);
  // strict parity mode (KMCUDA_B200_STRICT_UPDATE=1): the reference's running-sum update in sample order, in place
  KMCUDAResult update_reference_order(uint32_t n, const float* X, const uint32_t* assignments, const uint32_t* prev,
                                      float* C, uint32_t* ccounts, cudaStream_t st);
  // after the stream has been synchronised: kmcudaRuntimeError if the tensor-core pipeline of the last pass
  // reported a timed-out barrier (its results are not valid), kmcudaSuccess otherwise
  KMCUDAResult check_pipeline();

  const int metric, device;
  const uint32_t max_n;
  const int D;
  const uint32_t K;
  const int verbosity;

  bool last_tc = false;
  uint32_t last_rechecked = 0, last_overflowed = 0;
  bool force_exact = false;  // KMCUDA_B200_FORCE_EXACT=1 (debug / parity tests)
  // KMCUDA_B200_GRAPH=1: the ~13 launches of an assignment pass are captured once per (buffers, n, stream) and replayed
  // as ONE CUDA graph launch (iterative runs call assign() with the same buffers; the centroids change in place)
  bool use_graph = false;
  cudaGraphExec_t assign_graph = nullptr;
  struct GraphKey {
    const float* X = nullptr;
    const float* C = nullptr;
    uint32_t* a = nullptr;
    uint32_t* prev = nullptr;
    uint32_t* ch = nullptr;
    uint32_t n = 0;
    cudaStream_t st = nullptr;
    bool operator==(const GraphKey& o) const {
      return X == o.X && C == o.C && a == o.a && prev == o.prev && ch == o.ch && n == o.n && st == o.st;
    }
  } graph_key;
  bool strict_update = false;  // KMCUDA_B200_STRICT_UPDATE=1
  DevBuf<uint32_t> su_keys_in, su_vals_in, su_keys_out, su_vals_out, su_offsets;
  DevBuf<char> su_cub;
  size_t su_cub_bytes = 0;

  // scratch
  DevBuf<float> csq;
  DevBuf<uint32_t> result;
  UpdateWorkspace ws;
  DevBuf<uint32_t> ws_keys_out, ws_vals_in, ws_vals_out, ws_offsets;
  DevBuf<uint32_t> d_count;   // assign_rows on the exact route: the list length
  DevBuf<float> ws_partial;
  DevBuf<float> ws_partial_w;   // weighted update only, allocated on first use
  DevBuf<float> prev_sums;   // cosine update: member sums of the previous iteration
  DevBuf<char> ws_cub;
  TcPlan* tc = nullptr;   // the tensor-core passes (Lloyd, Yinyang, mini-batch); nullptr: the exact kernels

  // Yinyang state (per shard)
  uint32_t G = 0;
  DevBuf<float> bounds, drift, maxdrift, oldC;
  DevBuf<uint32_t> passed, groups;
  DevBuf<uint32_t> yy_counters;      // [0] rows needing the exact upper bound, [1] rows passed to the local step
  DevBuf<float> yy_minlb, yy_tight_score;
  DevBuf<uint32_t> yy_tight_rows, yy_tight_cand, yy_gsize;
};

}  // namespace kmb
