// exchange.cu -- the centroid update's exchange step for ONE PROCESS PER GPU, over peer memory.
//
// The reference is single-process: after kmeans_adjust every GPU copies its centroid slice to the others with
// cudaMemcpyPeerAsync (reference src/kmeans.cu:980-990,1014-1024).  With one process per GPU (torchrun / MPI ranks) the
// sample shards live in different address spaces; the only data that has to cross is the [K][D] fp32 partial sums
// and the [K] member counts of every shard.  An NCCL all-reduce of that 1 MB is latency-bound (two collectives,
// ~0.12 ms at 8 GPUs); here every rank maps its peers' partial-sum buffers through CUDA IPC once, and per iteration
// ONE kernel per GPU
//   * publishes "my partial sums of iteration i are complete" with a system-scope store into every peer's flag row
//     (over NVLink / NVSwitch),
//   * waits for the same flag from every peer (a bounded spin: a dead peer becomes kmcudaRuntimeError, not a hang),
//   * reads every peer's sums straight from the peer's HBM with 16-byte loads and adds them IN RANK ORDER, so all ranks
//     hold bit-identical totals (an NCCL ring / tree does not promise that).
// The partial buffers are double-buffered by iteration parity, which makes a "reads complete" handshake unnecessary:
// a peer can only start overwriting buffer (i & 1) in iteration i + 2, after it has seen this rank's flag of
// iteration i + 1, which this rank's stream sends after its reduce kernel of iteration i has finished.
#include <cuda_runtime.h>

#include <algorithm>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <new>

#include "kernels.h"
#include "kmcuda_b200.h"
#include "shard.h"

namespace kmb {

constexpr int kMaxRanks = 32;
constexpr long long kExchangeTimeoutCycles = 40000000000ll;   // ~20 s at 2 GHz: a peer that never arrives

struct ExchangePeers {
  char* base[kMaxRanks];
  int n, rank;
};

__device__ __forceinline__ uint32_t ld_acquire_sys(const uint32_t* p) {
  uint32_t v;
  asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void st_release_sys(uint32_t* p, uint32_t v) {
  asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ float4 ld_sys_f4(const float4* p) {
  float4 v;
  asm volatile("ld.relaxed.sys.global.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ float ld_sys_f(const float* p) {
  float v;
  asm volatile("ld.relaxed.sys.global.f32 %0, [%1];" : "=f"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ uint32_t ld_sys_u(const uint32_t* p) {
  uint32_t v;
  asm volatile("ld.relaxed.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}

__global__ void __launch_bounds__(256)
exchange_reduce_kernel(const ExchangePeers pp, size_t off_sums, size_t off_counts, size_t off_flags, uint32_t iter,
                       size_t nvec4, size_t nsums, uint32_t K, float* __restrict__ out_sums,
                       uint32_t* __restrict__ out_counts, uint32_t* err) {
  __shared__ int s_fail;
  // an earlier exchange of this handle timed out: the ranks are out of step for good, do not wait another 20 s per launch
  if (ld_acquire_sys(err) != 0u) return;
  if (threadIdx.x == 0) s_fail = 0;
  // (the partial sums were written by earlier kernels of this stream: complete and visible before this kernel started)
  if (blockIdx.x == 0 && threadIdx.x < pp.n)
    st_release_sys(reinterpret_cast<uint32_t*>(pp.base[threadIdx.x] + off_flags) + pp.rank, iter);
  __syncthreads();
  if (threadIdx.x < pp.n) {
    const uint32_t* f = reinterpret_cast<const uint32_t*>(pp.base[pp.rank] + off_flags) + threadIdx.x;
    const long long t0 = clock64();
    while (static_cast<int32_t>(ld_acquire_sys(f) - iter) < 0) {
      __nanosleep(64);
      if (clock64() - t0 > kExchangeTimeoutCycles) {
        s_fail = 1;
        break;
      }
    }
  }
  __syncthreads();
  if (s_fail) {
    if (threadIdx.x == 0) atomicExch(err, 1u);
    return;
  }
  const size_t stride = static_cast<size_t>(gridDim.x) * blockDim.x;
  const size_t t = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  for (size_t i = t; i < nvec4; i += stride) {
    float4 acc = ld_sys_f4(reinterpret_cast<const float4*>(pp.base[0] + off_sums) + i);
    for (int d = 1; d < pp.n; d++) {
      const float4 v = ld_sys_f4(reinterpret_cast<const float4*>(pp.base[d] + off_sums) + i);
      acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
    }
    reinterpret_cast<float4*>(out_sums)[i] = acc;
  }
  for (size_t i = nvec4 * 4 + t; i < nsums; i += stride) {
    float acc = ld_sys_f(reinterpret_cast<const float*>(pp.base[0] + off_sums) + i);
    for (int d = 1; d < pp.n; d++) acc += ld_sys_f(reinterpret_cast<const float*>(pp.base[d] + off_sums) + i);
    out_sums[i] = acc;
  }
  for (size_t c = t; c < K; c += stride) {
    uint32_t acc = 0;   // exact integer sum (counts never go through fp32)
    for (int d = 0; d < pp.n; d++) acc += ld_sys_u(reinterpret_cast<const uint32_t*>(pp.base[d] + off_counts) + c);
    out_counts[c] = acc;
  }
}

}  // namespace kmb

struct kmcuda_b200_exchange {
  int rank = 0, world = 1, device = 0;
  uint32_t K = 0;
  int D = 0;
  size_t off_sums[2] = {0, 0}, off_counts[2] = {0, 0}, off_flags = 0, off_err = 0, bytes = 0;
  char* local = nullptr;
  char* peer[kmb::kMaxRanks] = {};
  bool opened[kmb::kMaxRanks] = {};
  bool connected = false;
  uint32_t iter = 0;
  uint32_t* h_err = nullptr;   // pinned copy of the error word
};

extern "C" {

uint32_t kmcuda_b200_exchange_handle_bytes(void) { return static_cast<uint32_t>(sizeof(cudaIpcMemHandle_t)); }

KMCUDAResult kmcuda_b200_exchange_create(kmcuda_b200_exchange** out, uint32_t clusters_size, uint16_t features_size,
                                         int32_t rank, int32_t world, void* handle_out) {
  if (!out || !handle_out || clusters_size < 2 || features_size == 0 || world < 1 || world > kmb::kMaxRanks || rank < 0 ||
      rank >= world)
    return kmcudaInvalidArguments;
  auto* ex = new (std::nothrow) kmcuda_b200_exchange;
  if (!ex) return kmcudaMemoryAllocationFailure;
  ex->rank = rank;
  ex->world = world;
  ex->K = clusters_size;
  ex->D = features_size;
  if (cudaGetDevice(&ex->device) != cudaSuccess) { delete ex; return kmcudaNoSuchDevice; }
  auto align = [](size_t v) { return (v + 255) / 256 * 256; };
  const size_t sums_bytes = align(static_cast<size_t>(ex->K) * ex->D * sizeof(float));
  const size_t counts_bytes = align(static_cast<size_t>(ex->K) * sizeof(uint32_t));
  size_t o = 0;
  ex->off_sums[0] = o; o += sums_bytes;
  ex->off_sums[1] = o; o += sums_bytes;
  ex->off_counts[0] = o; o += counts_bytes;
  ex->off_counts[1] = o; o += counts_bytes;
  ex->off_flags = o; o += 256;
  ex->off_err = o; o += 256;
  ex->bytes = o;
  // a dedicated cudaMalloc block (not the workspace cache): the IPC handle exports the whole allocation
  if (cudaMalloc(reinterpret_cast<void**>(&ex->local), ex->bytes) != cudaSuccess) {
    cudaGetLastError();
    delete ex;
    return kmcudaMemoryAllocationFailure;
  }
  cudaIpcMemHandle_t h;
  if (cudaMemset(ex->local, 0, ex->bytes) != cudaSuccess || cudaDeviceSynchronize() != cudaSuccess ||
      cudaIpcGetMemHandle(&h, ex->local) != cudaSuccess ||
      cudaHostAlloc(reinterpret_cast<void**>(&ex->h_err), sizeof(uint32_t), cudaHostAllocPortable) != cudaSuccess) {
    cudaGetLastError();
    cudaFree(ex->local);
    delete ex;
    return kmcudaRuntimeError;
  }
  *ex->h_err = 0;
  memcpy(handle_out, &h, sizeof(h));
  ex->peer[rank] = ex->local;
  *out = ex;
  return kmcudaSuccess;
}

/* all_handles: world * kmcuda_b200_exchange_handle_bytes() bytes, rank-major (what an all-gather of the handles gives) */
KMCUDAResult kmcuda_b200_exchange_connect(kmcuda_b200_exchange* ex, const void* all_handles) {
  if (!ex || !all_handles) return kmcudaInvalidArguments;
  if (cudaSetDevice(ex->device) != cudaSuccess) return kmcudaNoSuchDevice;
  const char* hs = static_cast<const char*>(all_handles);
  for (int r = 0; r < ex->world; r++) {
    if (r == ex->rank) continue;
    cudaIpcMemHandle_t h;
    memcpy(&h, hs + static_cast<size_t>(r) * sizeof(h), sizeof(h));
    void* p = nullptr;
    cudaError_t e = cudaIpcOpenMemHandle(&p, h, cudaIpcMemLazyEnablePeerAccess);
    if (e != cudaSuccess) {
      fprintf(stderr, "[kmcuda_b200] cudaIpcOpenMemHandle(rank %d) failed on rank %d: %s\n", r, ex->rank, cudaGetErrorString(e));
      cudaGetLastError();
      return kmcudaRuntimeError;
    }
    ex->peer[r] = static_cast<char*>(p);
    ex->opened[r] = true;
  }
  ex->connected = true;
  return kmcudaSuccess;
}

/* Where this iteration's partial sums / counts go (device pointers into the exported block); the pair alternates
 * between two buffers from call to call of kmcuda_b200_exchange_reduce(). */
KMCUDAResult kmcuda_b200_exchange_buffers(kmcuda_b200_exchange* ex, float** sums, uint32_t** counts) {
  if (!ex || !sums || !counts) return kmcudaInvalidArguments;
  const int b = static_cast<int>((ex->iter + 1) & 1u);
  *sums = reinterpret_cast<float*>(ex->local + ex->off_sums[b]);
  *counts = reinterpret_cast<uint32_t*>(ex->local + ex->off_counts[b]);
  return kmcudaSuccess;
}

/* total_sums [K][D], total_counts [K] (device, this rank) = sum over ranks, in rank order, of the buffers that
 * kmcuda_b200_exchange_buffers() handed out for this iteration.  Enqueued on `stream`; every rank must call it once per
 * iteration. */
KMCUDAResult kmcuda_b200_exchange_reduce(kmcuda_b200_exchange* ex, float* total_sums, uint32_t* total_counts,
                                         void* stream) {
  if (!ex || !total_sums || !total_counts || !ex->connected) return kmcudaInvalidArguments;
  if (*ex->h_err) return kmcudaRuntimeError;   // an earlier exchange timed out: the peers are out of step
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  ex->iter++;
  const int b = static_cast<int>(ex->iter & 1u);
  kmb::ExchangePeers pp;
  pp.n = ex->world;
  pp.rank = ex->rank;
  for (int r = 0; r < ex->world; r++) pp.base[r] = ex->peer[r];
  const size_t nsums = static_cast<size_t>(ex->K) * ex->D;
  const size_t nvec4 = nsums / 4;
  const unsigned grid = static_cast<unsigned>(std::min<size_t>(kmb::device_sms(), (nvec4 + 255) / 256 + 1));
  uint32_t* d_err = reinterpret_cast<uint32_t*>(ex->local + ex->off_err);
  kmb::exchange_reduce_kernel<<<grid, 256, 0, st>>>(pp, ex->off_sums[b], ex->off_counts[b], ex->off_flags, ex->iter,
                                                     nvec4, nsums, ex->K, total_sums, total_counts, d_err);
  if (cudaGetLastError() != cudaSuccess) return kmcudaRuntimeError;
  if (cudaMemcpyAsync(ex->h_err, d_err, sizeof(uint32_t), cudaMemcpyDeviceToHost, st) != cudaSuccess) return kmcudaRuntimeError;
  return kmcudaSuccess;
}

/* 0 = every exchange so far completed; non-zero = a peer never arrived (valid after `stream` was synchronised) */
uint32_t kmcuda_b200_exchange_error(kmcuda_b200_exchange* ex) { return ex && ex->h_err ? *ex->h_err : 1u; }

/* Call after a barrier of the ranks (no peer may still be reading this rank's block). */
void kmcuda_b200_exchange_destroy(kmcuda_b200_exchange* ex) {
  if (!ex) return;
  cudaSetDevice(ex->device);
  cudaDeviceSynchronize();
  for (int r = 0; r < ex->world; r++)
    if (ex->opened[r]) cudaIpcCloseMemHandle(ex->peer[r]);
  if (ex->local) cudaFree(ex->local);
  if (ex->h_err) cudaFreeHost(ex->h_err);
  cudaGetLastError();
  delete ex;
}

}  // extern "C"
