// transfer.cu -- the copy routes between the caller's memory (host, or one device) and the devices of a call: the staged
// ingest of pageable host memory, copy_in / copy_out (job.h) and the end of a device's stream.
#include <mutex>
#include <thread>

#include "job.h"

namespace kmb {

// ------------------------------------------------------------------------------------------------
// Ingest of PAGEABLE host memory (SURVEY.md 8f-2; the reference: one pageable cudaMemcpy of the whole matrix to every
// GPU, kmcuda.cc:139-170).  A pageable cudaMemcpyAsync is staged by the driver through one small pinned buffer by one
// thread: ~11 GB/s on this box, 0.72 s of a 1.2 s C2 run.  Here a few host threads copy interleaved 16 MB chunks into
// their own pinned staging buffers (kept for the life of the process) and enqueue the DMA on their own streams, so the
// page-touching memcpy of one chunk overlaps the DMA of the others.  Pinned or registered sources, small copies and
// KMCUDA_B200_INGEST_THREADS=1 take the plain cudaMemcpyAsync.
// ------------------------------------------------------------------------------------------------
struct IngestLane {
  int dev = -1;
  cudaStream_t st = nullptr;
  void* buf[2] = {nullptr, nullptr};
  cudaEvent_t ev[2] = {nullptr, nullptr};
};
static constexpr size_t kIngestChunk = 16u << 20;
static std::vector<IngestLane>& ingest_lanes() {
  static std::vector<IngestLane> lanes;
  return lanes;
}
static bool ingest_lane_ready(IngestLane& l, int dev) {
  if (l.dev == dev && l.st) return true;
  if (cudaSetDevice(dev) != cudaSuccess) return false;
  if (l.st) {   // the lane belonged to another device: rebuild its stream and events there
    cudaStreamDestroy(l.st);
    for (int i = 0; i < 2; i++) cudaEventDestroy(l.ev[i]);
    l.st = nullptr;
  }
  if (cudaStreamCreateWithFlags(&l.st, cudaStreamNonBlocking) != cudaSuccess) { l.st = nullptr; return false; }
  for (int i = 0; i < 2; i++) {
    if (!l.buf[i] && cudaHostAlloc(&l.buf[i], kIngestChunk, cudaHostAllocPortable) != cudaSuccess) { l.buf[i] = nullptr; return false; }
    if (cudaEventCreateWithFlags(&l.ev[i], cudaEventDisableTiming) != cudaSuccess) return false;
  }
  l.dev = dev;
  return true;
}
// copies `bytes` from host `src` to device `dst` (current device `dev`); returns when the data is on the device or
// enqueued on `st` (plain path); cudaSuccess or the first error
static cudaError_t host_to_device(void* dst, const void* src, size_t bytes, int dev, cudaStream_t st) {
  int nthreads = 6;
  if (const char* e = getenv("KMCUDA_B200_INGEST_THREADS")) nthreads = std::max(1, std::min(16, atoi(e)));
  bool pageable = false;
  if (bytes >= (256u << 20) && nthreads > 1) {   // (below that the one-time cost of the pinned staging buffers, ~50 ms, is not earned back)
    cudaPointerAttributes at;
    if (cudaPointerGetAttributes(&at, src) == cudaSuccess) pageable = at.type == cudaMemoryTypeUnregistered;
    else cudaGetLastError();
  }
  if (!pageable) return cudaMemcpyAsync(dst, src, bytes, cudaMemcpyHostToDevice, st);
  static std::mutex mu;                       // knn_cuda drives several devices from concurrent host threads: the lanes
  std::lock_guard<std::mutex> lock(mu);       // (staging buffers) are shared, one staged copy at a time
  auto& lanes = ingest_lanes();
  if (static_cast<int>(lanes.size()) < nthreads) lanes.resize(nthreads);
  for (int t = 0; t < nthreads; t++)
    if (!ingest_lane_ready(lanes[t], dev)) {
      cudaGetLastError();
      return cudaMemcpyAsync(dst, src, bytes, cudaMemcpyHostToDevice, st);
    }
  const size_t nchunks = (bytes + kIngestChunk - 1) / kIngestChunk;
  std::vector<cudaError_t> err(nthreads, cudaSuccess);
  std::vector<std::thread> workers;
  for (int t = 0; t < nthreads; t++)
    workers.emplace_back([&, t]() {
      IngestLane& l = lanes[t];
      if ((err[t] = cudaSetDevice(dev)) != cudaSuccess) return;
      int slot = 0;
      for (size_t c = t; c < nchunks; c += nthreads, slot ^= 1) {
        const size_t off = c * kIngestChunk, len = std::min(kIngestChunk, bytes - off);
        if ((err[t] = cudaEventSynchronize(l.ev[slot])) != cudaSuccess) return;   // the DMA that last read this buffer
        memcpy(l.buf[slot], static_cast<const char*>(src) + off, len);
        if ((err[t] = cudaMemcpyAsync(static_cast<char*>(dst) + off, l.buf[slot], len, cudaMemcpyHostToDevice, l.st)) != cudaSuccess) return;
        if ((err[t] = cudaEventRecord(l.ev[slot], l.st)) != cudaSuccess) return;
      }
      err[t] = cudaStreamSynchronize(l.st);
    });
  for (auto& w : workers) w.join();
  for (int t = 0; t < nthreads; t++)
    if (err[t] != cudaSuccess) return err[t];
  return cudaSuccess;
}

// the raw copy of `bytes` from the caller's `src` into `dst` on device `dev`
static cudaError_t copy_bytes_in(void* dst, const void* src, size_t bytes, int dev, int device_ptrs, bool staged,
                                 cudaStream_t st) {
  if (device_ptrs >= 0) return cudaMemcpyPeerAsync(dst, dev, src, device_ptrs, bytes, st);
  if (staged) return host_to_device(dst, src, bytes, dev, st);
  return cudaMemcpyAsync(dst, src, bytes, cudaMemcpyHostToDevice, st);
}

template <typename T>
KMCUDAResult copy_in(DevBuf<T>& dst, const T* src, size_t count, int dev, int device_ptrs, bool fp16x2, cudaStream_t st,
                     int verbosity, bool borrow, bool staged) {
  if (!fp16x2 && borrow && device_ptrs == dev) {
    dst.borrow(const_cast<T*>(src));   // work in place, read-only
    return kmcudaSuccess;
  }
  KMB_CU(dst.alloc(count), kmcudaMemoryAllocationFailure);
  if (!fp16x2) {
    KMB_CU(copy_bytes_in(dst.get(), src, count * sizeof(T), dev, device_ptrs, staged, st), kmcudaMemoryCopyError);
    return kmcudaSuccess;
  }
  DevBuf<char> tmp;
  const void* hsrc = src;
  if (!borrow || device_ptrs != dev) {
    KMB_CU(tmp.alloc(count * 2), kmcudaMemoryAllocationFailure);
    KMB_CU(copy_bytes_in(tmp.get(), src, count * 2, dev, device_ptrs, staged, st), kmcudaMemoryCopyError);
    hsrc = tmp.get();
  }
  const cudaError_t widened = launch_half_to_float(hsrc, reinterpret_cast<float*>(dst.get()), count, st);
  const cudaError_t synced = cudaStreamSynchronize(st);   // tmp dies here, also after a failed launch
  KMB_CU(widened, kmcudaRuntimeError);
  KMB_CU(synced, kmcudaMemoryCopyError);
  return kmcudaSuccess;
}
template KMCUDAResult copy_in(DevBuf<float>&, const float*, size_t, int, int, bool, cudaStream_t, int, bool, bool);
template KMCUDAResult copy_in(DevBuf<uint32_t>&, const uint32_t*, size_t, int, int, bool, cudaStream_t, int, bool, bool);

template <typename T>
KMCUDAResult copy_out(T* dst, const T* src, size_t count, int dev, int device_ptrs, bool fp16x2, cudaStream_t st,
                      int verbosity) {
  DevBuf<char> tmp;
  const void* dsrc = src;
  if (fp16x2) {
    KMB_CU(tmp.alloc(count * 2), kmcudaMemoryAllocationFailure);
    KMB_CU(launch_float_to_half(reinterpret_cast<const float*>(src), tmp.get(), count, st), kmcudaRuntimeError);
    dsrc = tmp.get();
  }
  const size_t bytes = fp16x2 ? count * 2 : count * sizeof(T);
  const cudaError_t copied = device_ptrs < 0 ? cudaMemcpyAsync(dst, dsrc, bytes, cudaMemcpyDeviceToHost, st)
                                             : cudaMemcpyPeerAsync(dst, device_ptrs, dsrc, dev, bytes, st);
  const cudaError_t synced = fp16x2 ? cudaStreamSynchronize(st) : cudaSuccess;   // tmp dies here
  KMB_CU(copied, kmcudaMemoryCopyError);
  KMB_CU(synced, kmcudaMemoryCopyError);
  return kmcudaSuccess;
}
template KMCUDAResult copy_out(float*, const float*, size_t, int, int, bool, cudaStream_t, int);
template KMCUDAResult copy_out(uint32_t*, const uint32_t*, size_t, int, int, bool, cudaStream_t, int);

void sync_stream(int dev, cudaStream_t st) {
  if (!st) return;
  cudaSetDevice(dev);
  cudaStreamSynchronize(st);
}

void retire_stream(int dev, cudaStream_t st, std::initializer_list<cudaEvent_t> events) {
  if (!st) return;
  sync_stream(dev, st);
  for (cudaEvent_t ev : events)
    if (ev) cudaEventDestroy(ev);
  cudaStreamDestroy(st);
}

}  // namespace kmb
