// api.cu -- kmeans_cuda() / knn_cuda(): the drop-in C ABI of include/kmcuda.h.
//
// Role of the reference's kmcuda.cc (argument validation kmcuda.cc:19-61, device mask -> device list
// :63-137, allocation + ingest :139-170, centroid initialisation :189-400, driver :402-531, k-NN
// driver :572-730) and of the host halves of kmeans.cu (Lloyd loop :934-1026, Yinyang loop
// :1028-1263).  Differences by design (DESIGN.md): samples are range-partitioned across the GPUs in
// the mask instead of replicated; no transpose; the per-iteration exchange is ONE NCCL all-reduce of
// the [K][D] partial sums + [K] counts instead of 5-6 rounds of peer copies; centroid update is a
// deterministic sort + segmented compensated sum instead of one thread per centroid.
#include <dlfcn.h>
#include <nccl.h>  // types and enums only: NCCL is bound at run time, see NcclApi below

#include <algorithm>
#include <cinttypes>
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <memory>
#include <chrono>
#include <map>
#include <mutex>
#include <random>
#include <string>
#include <thread>
#include <atomic>
#include <utility>
#include <vector>

#include "kmcuda.h"
#include "kmcuda_b200.h"
#include "shard.h"

namespace kmb {

static const float kYinyangGroupTolerance = 0.02f;      // reference kmeans.cu:27
static const float kYinyangDraftReassignments = 0.11f;  // reference kmeans.cu:28
static const float kYinyangRefreshEpsilon = 1e-4f;      // reference kmeans.cu:29
static const uint32_t kKMeansParallelRounds = 5;        // k-means|| rounds when init_params gives none
static const uint32_t kKMeansParallelMaxRounds = 32;    // the round number is 8 bits of the draw hash's key

// NCCL is resolved lazily with dlopen the first time a job spans more than one GPU.  Linking it
// would either pin a second libnccl.so.2 into processes that also import torch (which ships its own,
// newer NCCL under the same soname) or, linked statically, add ~400 MB to the library.
struct NcclApi {
  ncclResult_t (*CommInitAll)(ncclComm_t*, int, const int*) = nullptr;
  ncclResult_t (*CommDestroy)(ncclComm_t) = nullptr;
  ncclResult_t (*AllReduce)(const void*, void*, size_t, ncclDataType_t, ncclRedOp_t, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*GroupStart)() = nullptr;
  ncclResult_t (*GroupEnd)() = nullptr;
  const char* (*GetErrorString)(ncclResult_t) = nullptr;
  bool ok = false;
};

static const NcclApi& nccl_api() {
  static NcclApi api;
  static bool tried = false;
  if (!tried) {
    tried = true;
    void* h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_NOLOAD | RTLD_LOCAL);  // already in the process?
    if (!h) h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_LOCAL);
    if (!h) h = dlopen("libnccl.so", RTLD_NOW | RTLD_LOCAL);
    if (h) {
      api.CommInitAll = reinterpret_cast<decltype(api.CommInitAll)>(dlsym(h, "ncclCommInitAll"));
      api.CommDestroy = reinterpret_cast<decltype(api.CommDestroy)>(dlsym(h, "ncclCommDestroy"));
      api.AllReduce = reinterpret_cast<decltype(api.AllReduce)>(dlsym(h, "ncclAllReduce"));
      api.GroupStart = reinterpret_cast<decltype(api.GroupStart)>(dlsym(h, "ncclGroupStart"));
      api.GroupEnd = reinterpret_cast<decltype(api.GroupEnd)>(dlsym(h, "ncclGroupEnd"));
      api.GetErrorString = reinterpret_cast<decltype(api.GetErrorString)>(dlsym(h, "ncclGetErrorString"));
      api.ok = api.CommInitAll && api.CommDestroy && api.AllReduce && api.GroupStart && api.GroupEnd &&
               api.GetErrorString;
    }
  }
  return api;
}

// NCCL communicators (fallback exchange, see Job::update) are cached per device list for the life of the process:
// ncclCommInitAll costs seconds to minutes and the library is not re-entrant anyway (kmcuda.h:25-26)
static std::map<std::vector<int>, std::vector<ncclComm_t>>& comm_cache() {
  static std::map<std::vector<int>, std::vector<ncclComm_t>> cache;
  return cache;
}
static void drop_cached_comms() {
  for (auto& kv : comm_cache())
    for (ncclComm_t c : kv.second)
      if (c) nccl_api().CommDestroy(c);
  comm_cache().clear();
}

struct Dev {
  int dev = 0;
  cudaStream_t st = nullptr;
  uint32_t off = 0, len = 0;
  std::unique_ptr<Shard> shard;
  DevBuf<float> X, C, sums, dists;
  DevBuf<float> rsums;           // multi-GPU: the shard sums reduced over all devices (peer loads, fixed order)
  DevBuf<uint32_t> rcounts;
  DevBuf<uint32_t> assign, prev, ccounts, counts, d_changed;
  DevBuf<double> d_dsum;
  // sample weights (weighted jobs only): this shard's slice, the per-cluster weight totals of the shard (wsums), of all
  // shards (rweights, peer exchange) and of the previous update (cweights, the cosine recurrence's old count)
  DevBuf<float> w, wsums, rweights, cweights;
  cudaEvent_t ev_partial = nullptr;   // this device's partial sums are complete
  cudaEvent_t ev_reduced = nullptr;   // this device has finished reading every peer's partial sums
  ncclComm_t comm = nullptr;
};

// equal split of `amount` rows over the devices, chunk starts aligned to 512 bytes without
// breaking rows (same rule as the reference's distribute(), private.h:240-273)
std::vector<std::pair<uint32_t, uint32_t>> split_rows(uint32_t amount, uint32_t row_bytes, size_t ndev) {
  std::vector<std::pair<uint32_t, uint32_t>> res;
  if (ndev == 0) return res;
  if (ndev == 1) {
    res.emplace_back(0, amount);
    return res;
  }
  uint32_t a = row_bytes, b = 512, gcd = 0;
  for (;;) {
    if (a == 0) { gcd = b; break; }
    b %= a;
    if (b == 0) { gcd = a; break; }
    a %= b;
  }
  uint32_t stride = 512 / gcd, offset = 0;
  for (size_t i = 0; i + 1 < ndev; i++) {
    float step = (amount - offset + .0f) / (ndev - i);
    uint32_t len = static_cast<uint32_t>(roundf(step / stride)) * stride;
    len = std::min(len, amount - offset);
    res.emplace_back(offset, len);
    offset += len;
  }
  res.emplace_back(offset, amount - offset);
  return res;
}

static KMCUDAResult list_devices(uint32_t device, int verbosity, std::vector<int>* devs) {
  int count = 0;
  if (cudaGetDeviceCount(&count) != cudaSuccess || count == 0) return kmcudaNoSuchDevice;
  if (count < 32 && device > (1u << count)) return kmcudaNoSuchDevice;  // kmcuda.cc:40-44
  if (device == 0) device = count >= 32 ? 0xFFFFFFFFu : (1u << count) - 1;
  for (int dev = 0; device; dev++, device >>= 1) {
    if (!(device & 1)) continue;
    if (dev >= count || cudaSetDevice(dev) != cudaSuccess) {
      KMB_INFO("failed to cudaSetDevice(%d)\n", dev);
      continue;
    }
    cudaDeviceProp props;
    if (cudaGetDeviceProperties(&props, dev) != cudaSuccess) continue;
    if (props.major != 9 || props.minor != 0) {   // sm_90a code runs on compute capability 9.0 only
      KMB_INFO("compute capability mismatch for device %d: this build targets sm_90a, have %d.%d\n",
               dev, props.major, props.minor);
      continue;
    }
    devs->push_back(dev);
  }
  return devs->empty() ? kmcudaNoSuchDevice : kmcudaSuccess;
}

static void enable_p2p(const std::vector<int>& devs, int extra, int verbosity) {
  std::vector<int> all(devs);
  if (extra >= 0 && std::find(all.begin(), all.end(), extra) == all.end()) all.push_back(extra);
  if (all.size() < 2) return;
  for (int d1 : all) {
    cudaSetDevice(d1);
    for (int d2 : all) {
      if (d1 == d2) continue;
      int access = 0;
      cudaDeviceCanAccessPeer(&access, d1, d2);
      if (!access) {
        KMB_INFO("warning: p2p %d <-> %d is impossible\n", d1, d2);
        continue;
      }
      cudaError_t e = cudaDeviceEnablePeerAccess(d2, 0);
      if (e == cudaErrorPeerAccessAlreadyEnabled) cudaGetLastError();
      else if (e != cudaSuccess) KMB_INFO("warning: failed to enable p2p on gpu #%d: %s\n", d1, cudaGetErrorString(e));
    }
  }
}

// Optional wall-clock phase profile (KMCUDA_B200_TIMING=1): every mark() synchronises the devices and books
// the time since the previous mark; the table goes to stderr when the call returns.  Off by default
// (no extra synchronisation).
struct PhaseProfile {
  bool on = false;
  std::vector<int> devs;
  std::vector<std::pair<std::string, double>> acc;
  std::chrono::steady_clock::time_point last;
  void begin(const std::vector<int>& d) {
    const char* e = getenv("KMCUDA_B200_TIMING");
    on = e && e[0] == '1';
    devs = d;
    acc.clear();
    last = std::chrono::steady_clock::now();
  }
  void mark(const char* name) {
    if (!on) return;
    for (int d : devs) { cudaSetDevice(d); cudaDeviceSynchronize(); }
    auto now = std::chrono::steady_clock::now();
    double ms = std::chrono::duration<double, std::milli>(now - last).count();
    last = now;
    for (auto& kv : acc) if (kv.first == name) { kv.second += ms; return; }
    acc.emplace_back(name, ms);
  }
  void report(const char* what) {
    if (!on) return;
    double tot = 0;
    for (auto& kv : acc) tot += kv.second;
    fprintf(stderr, "[kmcuda_b200 timing] %s: total %.2f ms\n", what, tot);
    for (auto& kv : acc) fprintf(stderr, "[kmcuda_b200 timing]   %-28s %10.2f ms\n", kv.first.c_str(), kv.second);
  }
};
static PhaseProfile g_prof;   // the library is not re-entrant (kmcuda.h:25-26), one profile is enough

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

class Job {
 public:
  Job(int metric, uint32_t N, int D, uint32_t K, int verbosity)
      : metric(metric), N(N), D(D), K(K), verbosity(verbosity) {}
  ~Job() {
    for (auto& d : devs) {
      cudaSetDevice(d.dev);
      d.comm = nullptr;   // owned by the per-process cache (Job::setup)
      d.shard.reset();
      if (d.ev_partial) cudaEventDestroy(d.ev_partial);
      if (d.ev_reduced) cudaEventDestroy(d.ev_reduced);
      if (d.st) cudaStreamDestroy(d.st);
    }
  }

  const int metric;
  const uint32_t N;
  const int D;
  const uint32_t K;
  const int verbosity;
  std::vector<Dev> devs;
  bool peer_exchange = false;   // multi-GPU update through peer memory (NVLink / NVSwitch) instead of NCCL
  bool weighted = false;        // per-sample weights (kmcuda_b200_kmeans_weighted); set before setup()
  double wtotal = 0;            // sum of the weights (check_weights)
  std::vector<float> host_w;    // host copy of the weights for the host-side seeding steps (load_host_weights)

  KMCUDAResult setup(const std::vector<int>& dev_ids, bool alloc_samples);
  KMCUDAResult ingest(const float* samples, const float* weights, int device_ptrs, bool fp16x2);
  KMCUDAResult check_weights();
  KMCUDAResult load_host_weights();
  KMCUDAResult sync_all();
  KMCUDAResult set_centroids_from_host(const float* hostC);
  KMCUDAResult fetch_row(uint32_t idx, float* host_row);
  KMCUDAResult init_centroids(KMCUDAInitMethod method, const void* init_params, uint32_t seed,
                              int device_ptrs, bool fp16x2, const float* user_centroids);
  KMCUDAResult draw_first_centroid(float* hostC, uint32_t* first_out);
  KMCUDAResult init_random();
  KMCUDAResult init_plusplus();
  KMCUDAResult init_afkmc2(uint32_t m, uint32_t seed);
  KMCUDAResult init_kmeans_parallel(uint32_t rounds, uint32_t seed);
  KMCUDAResult assign_pass(uint32_t* changed);
  KMCUDAResult update();
  KMCUDAResult lloyd(float tolerance, int* iter_out, uint32_t* changed_out);
  KMCUDAResult lloyd_continue(float tolerance, int iter);
  KMCUDAResult yinyang(float tolerance, uint32_t G);
  KMCUDAResult minibatch(uint32_t batch_size, uint64_t max_steps, float tolerance, uint32_t seed);
  double lloyd_iter_ms = 0;   // wall time of the fastest complete Lloyd iteration of this run (assign pass + update), 0 = none yet
  KMCUDAResult group_centroids(uint32_t G, std::vector<uint32_t>* groups);
  KMCUDAResult average_distance(float* out);
};

KMCUDAResult Job::setup(const std::vector<int>& dev_ids, bool alloc_samples) {
  auto plan = split_rows(N, static_cast<uint32_t>(D) * sizeof(float), dev_ids.size());
  devs.resize(dev_ids.size());
  for (size_t i = 0; i < dev_ids.size(); i++) {
    Dev& d = devs[i];
    d.dev = dev_ids[i];
    d.off = plan[i].first;
    d.len = plan[i].second;
    KMB_CU(cudaSetDevice(d.dev), kmcudaNoSuchDevice);
    KMB_CU(cudaStreamCreateWithFlags(&d.st, cudaStreamNonBlocking), kmcudaRuntimeError);
    if (alloc_samples) KMB_CU(d.X.alloc(static_cast<size_t>(d.len) * D), kmcudaMemoryAllocationFailure);
    KMB_CU(d.C.alloc(static_cast<size_t>(K) * D), kmcudaMemoryAllocationFailure);
    KMB_CU(d.sums.alloc(static_cast<size_t>(K) * D), kmcudaMemoryAllocationFailure);
    KMB_CU(d.assign.alloc(d.len), kmcudaMemoryAllocationFailure);
    KMB_CU(d.prev.alloc(d.len), kmcudaMemoryAllocationFailure);
    KMB_CU(d.ccounts.alloc(K), kmcudaMemoryAllocationFailure);
    KMB_CU(d.counts.alloc(K), kmcudaMemoryAllocationFailure);
    KMB_CU(d.d_changed.alloc(1), kmcudaMemoryAllocationFailure);
    KMB_CU(d.d_dsum.alloc(1), kmcudaMemoryAllocationFailure);
    if (weighted) {
      KMB_CU(d.wsums.alloc(K), kmcudaMemoryAllocationFailure);
      KMB_CU(d.cweights.alloc(K), kmcudaMemoryAllocationFailure);
    }
    g_prof.mark("setup: stream + job buffers");
    d.shard.reset(new Shard(metric, d.dev, d.len, D, K, verbosity));
    KMB_RET(d.shard->create(true));
    g_prof.mark("setup: shard workspace + tensor-core plan");
  }
  if (devs.size() > 1) {
    // Exchange step of the centroid update.  Preferred: every GPU reads its peers' partial sums straight from
    // peer memory (NVLink 5 / NVSwitch: K*D*4 bytes per peer, 1 MB at 1024 x 256) and adds them in device order,
    // so all GPUs hold bit-identical centroids and no communicator has to be bootstrapped (ncclCommInitAll took
    // ~100 s on the first multi-GPU call in round 1).  Fallback when some pair has no peer access, or
    // KMCUDA_B200_EXCHANGE=nccl: one grouped ncclAllReduce of sums + counts per iteration.
    const char* ex = getenv("KMCUDA_B200_EXCHANGE");
    peer_exchange = !(ex && strcmp(ex, "nccl") == 0);
    for (size_t i = 0; i < devs.size() && peer_exchange; i++)
      for (size_t j = 0; j < devs.size() && peer_exchange; j++) {
        if (i == j) continue;
        int access = 0;
        if (cudaDeviceCanAccessPeer(&access, devs[i].dev, devs[j].dev) != cudaSuccess || !access) peer_exchange = false;
      }
    if (peer_exchange) {
      for (auto& d : devs) {
        KMB_CU(cudaSetDevice(d.dev), kmcudaNoSuchDevice);
        KMB_CU(d.rsums.alloc(static_cast<size_t>(K) * D), kmcudaMemoryAllocationFailure);
        KMB_CU(d.rcounts.alloc(K), kmcudaMemoryAllocationFailure);
        if (weighted) KMB_CU(d.rweights.alloc(K), kmcudaMemoryAllocationFailure);
        KMB_CU(cudaEventCreateWithFlags(&d.ev_partial, cudaEventDisableTiming), kmcudaRuntimeError);
        KMB_CU(cudaEventCreateWithFlags(&d.ev_reduced, cudaEventDisableTiming), kmcudaRuntimeError);
      }
      KMB_DEBUG("centroid update exchange: peer memory, %zu devices\n", devs.size());
    } else {
      if (!nccl_api().ok) {
        KMB_INFO("multi-GPU jobs without full peer access need NCCL (libnccl.so.2), which could not be loaded\n");
        return kmcudaRuntimeError;
      }
      auto it = comm_cache().find(dev_ids);
      if (it == comm_cache().end()) {
        std::vector<ncclComm_t> comms(devs.size());
        ncclResult_t r = nccl_api().CommInitAll(comms.data(), static_cast<int>(devs.size()), dev_ids.data());
        if (r != ncclSuccess) {
          KMB_INFO("ncclCommInitAll failed: %s\n", nccl_api().GetErrorString(r));
          return kmcudaRuntimeError;
        }
        it = comm_cache().emplace(dev_ids, comms).first;
      }
      for (size_t i = 0; i < devs.size(); i++) devs[i].comm = it->second[i];
      KMB_DEBUG("centroid update exchange: NCCL all-reduce, %zu ranks\n", devs.size());
    }
  }
  if (verbosity > 1) {
    printf("plans: [");
    for (size_t i = 0; i < devs.size(); i++) printf("%s(%" PRIu32 ", %" PRIu32 ")", i ? ", " : "", devs[i].off, devs[i].len);
    printf("]\n");
  }
  return kmcudaSuccess;
}

KMCUDAResult Job::sync_all() {
  for (auto& d : devs) {
    KMB_CU(cudaSetDevice(d.dev), kmcudaRuntimeError);
    KMB_CU(cudaStreamSynchronize(d.st), kmcudaRuntimeError);
  }
  return kmcudaSuccess;
}

// samples: [N][D] fp32, or [N][D/2] half2 when fp16x2 (D is already the real dimension here); weights: [N] fp32 or
// nullptr, on the host or on device `device_ptrs` like the samples (always fp32)
KMCUDAResult Job::ingest(const float* samples, const float* weights, int device_ptrs, bool fp16x2) {
  const size_t elem = fp16x2 ? 2 : 4;
  for (auto& d : devs) {
    KMB_CU(cudaSetDevice(d.dev), kmcudaRuntimeError);
    if (weights) {
      const float* wsrc = weights + d.off;
      if (device_ptrs == d.dev) {
        d.w.borrow(const_cast<float*>(wsrc));   // read-only
      } else {
        KMB_CU(d.w.alloc(d.len), kmcudaMemoryAllocationFailure);
        if (device_ptrs < 0)
          KMB_CU(host_to_device(d.w.get(), wsrc, sizeof(float) * d.len, d.dev, d.st), kmcudaMemoryCopyError);
        else
          KMB_CU(cudaMemcpyPeerAsync(d.w.get(), d.dev, wsrc, device_ptrs, sizeof(float) * d.len, d.st),
                 kmcudaMemoryCopyError);
      }
    }
    const size_t count = static_cast<size_t>(d.len) * D;
    const char* src = reinterpret_cast<const char*>(samples) + static_cast<size_t>(d.off) * D * elem;
    if (!fp16x2) {
      if (device_ptrs < 0) {
        KMB_CU(host_to_device(d.X.get(), src, count * 4, d.dev, d.st), kmcudaMemoryCopyError);
      } else if (device_ptrs == d.dev) {
        d.X.borrow(const_cast<float*>(reinterpret_cast<const float*>(src)));  // work in place, read-only
      } else {
        KMB_CU(cudaMemcpyPeerAsync(d.X.get(), d.dev, src, device_ptrs, count * 4, d.st), kmcudaMemoryCopyError);
      }
    } else {
      DevBuf<char> tmp;
      const void* hsrc = src;
      if (!(device_ptrs >= 0 && device_ptrs == d.dev)) {
        KMB_CU(tmp.alloc(count * 2), kmcudaMemoryAllocationFailure);
        if (device_ptrs < 0)
          KMB_CU(host_to_device(tmp.get(), src, count * 2, d.dev, d.st), kmcudaMemoryCopyError);
        else
          KMB_CU(cudaMemcpyPeerAsync(tmp.get(), d.dev, src, device_ptrs, count * 2, d.st), kmcudaMemoryCopyError);
        hsrc = tmp.get();
      }
      KMB_CU(launch_half_to_float(hsrc, d.X.get(), count, d.st), kmcudaRuntimeError);
      KMB_CU(cudaStreamSynchronize(d.st), kmcudaMemoryCopyError);  // tmp dies here
    }
  }
  return sync_all();
}

// every weight finite and >= 0, their sum > 0: one pass over each shard's slice on its device, then one flag and one
// partial total per device come back (the same check for host and device weights)
KMCUDAResult Job::check_weights() {
  for (auto& d : devs) {
    KMB_CU(cudaSetDevice(d.dev), kmcudaRuntimeError);
    KMB_CU(cudaMemsetAsync(d.d_changed.get(), 0, sizeof(uint32_t), d.st), kmcudaRuntimeError);
    KMB_CU(cudaMemsetAsync(d.d_dsum.get(), 0, sizeof(double), d.st), kmcudaRuntimeError);
    KMB_CU(launch_check_weights(d.w, d.len, d.d_changed, d.d_dsum, d.st), kmcudaRuntimeError);
  }
  uint32_t bad = 0;
  double total = 0;
  for (auto& d : devs) {
    uint32_t flag = 0;
    double part = 0;
    KMB_CU(cudaSetDevice(d.dev), kmcudaRuntimeError);
    KMB_CU(cudaMemcpyAsync(&flag, d.d_changed.get(), sizeof(flag), cudaMemcpyDeviceToHost, d.st), kmcudaMemoryCopyError);
    KMB_CU(cudaMemcpyAsync(&part, d.d_dsum.get(), sizeof(part), cudaMemcpyDeviceToHost, d.st), kmcudaMemoryCopyError);
    KMB_CU(cudaStreamSynchronize(d.st), kmcudaRuntimeError);
    bad |= flag;
    total += part;
  }
  if (bad) {
    KMB_INFO("sample weights must be finite and >= 0\n");
    return kmcudaInvalidArguments;
  }
  if (!(total > 0)) {
    KMB_INFO("the sample weights sum to 0\n");
    return kmcudaInvalidArguments;
  }
  wtotal = total;
  return kmcudaSuccess;
}

// host copy of the weights, for the seeding steps that run on the host (first centroid, random init, AFK-MC2, the
// multi-GPU k-means++ walk); fetched once from the shards, so host and device inputs are served alike
KMCUDAResult Job::load_host_weights() {
  if (!weighted || !host_w.empty()) return kmcudaSuccess;
  host_w.resize(N);
  for (auto& d : devs) {
    KMB_CU(cudaSetDevice(d.dev), kmcudaRuntimeError);
    KMB_CU(cudaMemcpyAsync(host_w.data() + d.off, d.w.get(), sizeof(float) * d.len, cudaMemcpyDeviceToHost, d.st),
           kmcudaMemoryCopyError);
  }
  return sync_all();
}

// a seeding pick that landed on a zero-weight row moves to the next positive-weight row (the previous one at the end);
// the same rule as skip_zero_weight in simt_kernels.cu
static uint32_t skip_zero_weight_host(const std::vector<float>& w, uint32_t s) {
  if (w.empty() || w[s] > 0.f) return s;
  for (uint32_t u = s + 1; u < w.size(); u++)
    if (w[u] > 0.f) return u;
  for (uint32_t u = s; u-- > 0;)
    if (w[u] > 0.f) return u;
  return s;
}

KMCUDAResult Job::set_centroids_from_host(const float* hostC) {
  for (auto& d : devs) {
    KMB_CU(cudaSetDevice(d.dev), kmcudaRuntimeError);
    KMB_CU(cudaMemcpyAsync(d.C.get(), hostC, sizeof(float) * static_cast<size_t>(K) * D,
                           cudaMemcpyHostToDevice, d.st), kmcudaMemoryCopyError);
  }
  return sync_all();
}

KMCUDAResult Job::fetch_row(uint32_t idx, float* host_row) {
  for (auto& d : devs) {
    if (idx >= d.off && idx < d.off + d.len) {
      KMB_CU(cudaSetDevice(d.dev), kmcudaRuntimeError);
      KMB_CU(cudaMemcpy(host_row, d.X.get() + static_cast<size_t>(idx - d.off) * D, sizeof(float) * D,
                        cudaMemcpyDeviceToHost), kmcudaMemoryCopyError);
      return kmcudaSuccess;
    }
  }
  return kmcudaRuntimeError;
}

// identity permutation of N rows shuffled with rand() the way libstdc++'s std::random_shuffle does (kmcuda.cc:245-260)
static std::vector<uint32_t> random_order(uint32_t N) {
  std::vector<uint32_t> chosen(N);
  for (uint32_t s = 0; s < N; s++) chosen[s] = s;
  for (uint32_t i = 1; i < N; i++) {
    uint32_t j = static_cast<uint32_t>(rand() % (static_cast<int64_t>(i) + 1));
    if (i != j) std::swap(chosen[i], chosen[j]);
  }
  return chosen;
}

// K distinct random samples; same host RNG walk as the reference (kmcuda.cc:245-260).
// Weighted: the walk over the shuffled order skips rows of weight 0.
KMCUDAResult Job::init_random() {
  KMB_INFO("randomly picking initial centroids...\n");
  KMB_RET(load_host_weights());
  const std::vector<uint32_t> chosen = random_order(N);
  std::vector<float> hostC(static_cast<size_t>(K) * D);
  uint32_t c = 0;
  for (uint32_t s = 0; s < N && c < K; s++) {
    if (weighted && !(host_w[chosen[s]] > 0.f)) continue;
    KMB_RET(fetch_row(chosen[s], hostC.data() + static_cast<size_t>(c) * D));
    c++;
  }
  if (c < K) {
    KMB_INFO("random init: only %" PRIu32 " samples have a positive weight, %" PRIu32 " clusters\n", c, K);
    return kmcudaInvalidArguments;
  }
  return set_centroids_from_host(hostC.data());
}

// first centroid of k-means++ / AFK-MC2: rand() % N, re-drawn while the row is NaN (kmcuda.cc:270-276) or has weight 0
KMCUDAResult Job::draw_first_centroid(float* hostC, uint32_t* first_out) {
  KMB_RET(load_host_weights());
  uint32_t first_index;
  float smoke = NAN;
  do {
    first_index = rand() % N;
    if (weighted && !(host_w[first_index] > 0.f)) continue;   // (smoke stays NaN: draw again)
    std::vector<float> row(D);
    KMB_RET(fetch_row(first_index, row.data()));
    smoke = row[0];
    if (smoke == smoke) memcpy(hostC, row.data(), sizeof(float) * D);
  } while (smoke != smoke);
  *first_out = first_index;
  return kmcudaSuccess;
}

// k-means++ driven by the host RNG: reference kmcuda.cc:262-333 + kernel kmeans.cu:42-67.  Weighted: the draw is
// proportional to w * d (the reference's d, not d^2, times the weight)
KMCUDAResult Job::init_plusplus() {
  std::vector<float> hostC(static_cast<size_t>(K) * D);
  std::vector<float> host_dists(N);
  uint32_t first_index;
  KMB_RET(draw_first_centroid(hostC.data(), &first_index));
  KMB_INFO("performing kmeans++...\n");
  {
    const char* hp = getenv("KMCUDA_B200_HOST_PLUSPLUS");   // A/B: the reference-shaped host loop below
    if (devs.size() == 1 && !(hp && hp[0] == '1')) {
      // device-resident rounds: no D2H of the distances, no host walk, no H2D of the chosen row; the draws are the
      // reference's rand() sequence (one per round, kmcuda.cc:296)
      Dev& d = devs[0];
      KMB_CU(cudaSetDevice(d.dev), kmcudaRuntimeError);
      const uint32_t nb = (d.len + 255) / 256;
      DevBuf<double> bsum, bpre;
      DevBuf<uint32_t> chosen;
      KMB_CU(d.dists.alloc(d.len), kmcudaMemoryAllocationFailure);
      KMB_CU(bsum.alloc(static_cast<size_t>(nb) + 1), kmcudaMemoryAllocationFailure);
      KMB_CU(bpre.alloc(static_cast<size_t>(nb) + 1), kmcudaMemoryAllocationFailure);
      KMB_CU(chosen.alloc(K), kmcudaMemoryAllocationFailure);
      KMB_CU(cudaMemcpyAsync(d.C.get(), hostC.data(), sizeof(float) * D, cudaMemcpyHostToDevice, d.st), kmcudaMemoryCopyError);
      for (uint32_t i = 1; i < K; i++) {
        const double choice = ((rand() + .0) / RAND_MAX);
        KMB_CU(launch_plusplus_round(metric, d.X, d.len, D, d.C.get(), i, choice, d.dists, bsum, bpre, chosen, d.st,
                                     d.w.get()), kmcudaRuntimeError);
        if ((i & 255) == 0) KMB_CU(cudaStreamSynchronize(d.st), kmcudaRuntimeError);   // keep the launch queue shallow
      }
      KMB_CU(cudaStreamSynchronize(d.st), kmcudaRuntimeError);
      d.dists.release();
      return kmcudaSuccess;
    }
  }
  for (auto& d : devs) {
    KMB_CU(cudaSetDevice(d.dev), kmcudaRuntimeError);
    KMB_CU(d.dists.alloc(d.len), kmcudaMemoryAllocationFailure);
  }
  for (uint32_t i = 1; i < K; i++) {
    if (verbosity > 1 || (verbosity > 0 && (K < 100 || i % (K / 100) == 0))) {
      printf("\rstep %d", i);
      fflush(stdout);
    }
    double dist_sum = 0;
    for (auto& d : devs) {
      KMB_CU(cudaSetDevice(d.dev), kmcudaRuntimeError);
      float* cdst = d.C.get() + static_cast<size_t>(i - 1) * D;
      KMB_CU(cudaMemcpyAsync(cdst, hostC.data() + static_cast<size_t>(i - 1) * D, sizeof(float) * D,
                             cudaMemcpyHostToDevice, d.st), kmcudaMemoryCopyError);
      KMB_CU(cudaMemsetAsync(d.d_dsum.get(), 0, sizeof(double), d.st), kmcudaRuntimeError);
      KMB_CU(launch_plusplus_step(metric, d.X, d.len, D, cdst, i == 1, d.dists, d.d_dsum, d.st, d.w.get()),
             kmcudaRuntimeError);
      KMB_CU(cudaMemcpyAsync(host_dists.data() + d.off, d.dists.get(), sizeof(float) * d.len,
                             cudaMemcpyDeviceToHost, d.st), kmcudaMemoryCopyError);
    }
    for (auto& d : devs) {
      double part = 0;
      KMB_CU(cudaSetDevice(d.dev), kmcudaRuntimeError);
      KMB_CU(cudaMemcpyAsync(&part, d.d_dsum.get(), sizeof(double), cudaMemcpyDeviceToHost, d.st), kmcudaMemoryCopyError);
      KMB_CU(cudaStreamSynchronize(d.st), kmcudaRuntimeError);
      dist_sum += part;
    }
    if (weighted)   // the walk below runs over w * d, the mass the device summed (dists[] on the device keep d)
      for (uint32_t s = 0; s < N; s++) host_dists[s] *= host_w[s];
    if (dist_sum != dist_sum) KMB_INFO("\ninternal bug inside kmeans_init_centroids: dist_sum is NaN\n");
    double choice = ((rand() + .0) / RAND_MAX);
    uint32_t choice_approx = static_cast<uint32_t>(choice * N);
    double choice_sum = choice * dist_sum;
    uint32_t j;
    if (choice_approx < 100) {
      double s2 = 0;
      for (j = 0; j < N && s2 < choice_sum; j++) s2 += host_dists[j];
    } else {
      double s2 = 0;
      for (uint32_t t = 0; t < choice_approx; t++) s2 += host_dists[t];
      if (s2 < choice_sum) {
        for (j = choice_approx; j < N && s2 < choice_sum; j++) s2 += host_dists[j];
      } else {
        for (j = choice_approx; j > 1 && s2 >= choice_sum; j--) s2 -= host_dists[j];
        j++;
      }
    }
    if (j == 0 || j > N) {
      KMB_INFO("\ninternal bug in kmeans_init_centroids: j = %" PRIu32 "\n", j);
      j = std::min(std::max(j, 1u), N);
    }
    if (weighted) j = 1 + skip_zero_weight_host(host_w, j - 1);
    KMB_RET(fetch_row(j - 1, hostC.data() + static_cast<size_t>(i) * D));
  }
  for (auto& d : devs) d.dists.release();
  return set_centroids_from_host(hostC.data());
}

// AFK-MC2 (Bachem et al. 2016; reference kmcuda.cc:337-396, kernels kmeans.cu:69-212): proposal distribution
// q = 1/(2N) + d(x, c0)^2 / (2 sum d^2), then for every further centroid a Markov chain of length m over
// candidates drawn from q, accepting with probability min(1, (p'/q')/(p/q)) where p = squared distance to the
// nearest chosen centroid.  The reference draws candidates and acceptance thresholds with cuRAND on the device;
// here the chain is driven by a host generator seeded with `seed` (deterministic per seed; the reference's own q
// depends on float atomics, so its runs are only statistically reproducible as well).  The distance work (q and
// the candidates' nearest-centroid distances) runs on the shards that own the samples.
//
// Weighted: q = w / (2 W) + w d^2 / (2 sum w d^2) and p = w * (squared distance), so zero-weight rows are never drawn.
KMCUDAResult Job::init_afkmc2(uint32_t m, uint32_t seed) {
  std::vector<float> hostC(static_cast<size_t>(K) * D);
  std::vector<float> host_dists(N);
  uint32_t first_index;
  KMB_RET(draw_first_centroid(hostC.data(), &first_index));   // kmcuda.cc:346-353
  KMB_INFO("afkmc2: calculating q (c0 = %" PRIu32 ")... ", first_index);
  for (auto& d : devs) {
    KMB_CU(cudaSetDevice(d.dev), kmcudaRuntimeError);
    KMB_CU(d.dists.alloc(std::max<size_t>(d.len, 2 * static_cast<size_t>(m))), kmcudaMemoryAllocationFailure);
    KMB_CU(cudaMemcpyAsync(d.C.get(), hostC.data(), sizeof(float) * D, cudaMemcpyHostToDevice, d.st), kmcudaMemoryCopyError);
    KMB_CU(cudaMemsetAsync(d.d_dsum.get(), 0, sizeof(double), d.st), kmcudaRuntimeError);
    KMB_CU(launch_plusplus_step(metric, d.X, d.len, D, d.C.get(), 1, d.dists, d.d_dsum, d.st), kmcudaRuntimeError);
    KMB_CU(cudaMemcpyAsync(host_dists.data() + d.off, d.dists.get(), sizeof(float) * d.len, cudaMemcpyDeviceToHost, d.st),
           kmcudaMemoryCopyError);
  }
  KMB_RET(sync_all());
  std::vector<float> q(N);
  std::vector<double> cdf(N);
  {
    // (unweighted: w = 1 and W = N)
    const double W = weighted ? wtotal : static_cast<double>(N);
    double dsum = 0;
    for (uint32_t i = 0; i < N; i++) {
      const double d2 = static_cast<double>(host_dists[i]) * host_dists[i];
      if (d2 == d2) dsum += weighted ? host_w[i] * d2 : d2;
    }
    double acc = 0;
    for (uint32_t i = 0; i < N; i++) {
      double d2 = static_cast<double>(host_dists[i]) * host_dists[i];
      if (!(d2 == d2)) d2 = 0;
      const double wi = weighted ? host_w[i] : 1.0;
      const double qi = wi / (2.0 * W) + (dsum > 0 ? wi * d2 / (2.0 * dsum) : wi / (2.0 * W));
      q[i] = static_cast<float>(qi);
      acc += qi;
      cdf[i] = acc;
    }
  }
  KMB_INFO("done\n");
  std::mt19937_64 gen(seed);
  auto uniform = [&gen]() { return (static_cast<double>(gen() >> 11) + 0.5) * (1.0 / 9007199254740992.0); };
  std::vector<uint32_t> cand(m), local(m);
  std::vector<float> p_cand(m), rand_a(m);
  struct Scratch { DevBuf<uint32_t> rows; DevBuf<float> mind; std::vector<uint32_t> slots; std::vector<float> host; };
  std::vector<Scratch> sc(devs.size());
  for (size_t i = 0; i < devs.size(); i++) {
    KMB_CU(cudaSetDevice(devs[i].dev), kmcudaRuntimeError);
    KMB_CU(sc[i].rows.alloc(m), kmcudaMemoryAllocationFailure);
    KMB_CU(sc[i].mind.alloc(m), kmcudaMemoryAllocationFailure);
    sc[i].host.resize(m);
  }
  for (uint32_t k = 1; k < K; k++) {
    if (verbosity > 1 || (verbosity > 0 && (K < 100 || k % (K / 100) == 0))) {
      printf("\rstep %d", k);
      fflush(stdout);
    }
    for (uint32_t j = 0; j < m; j++) {   // kmeans_afkmc2_random_step: first index whose cumulative q reaches the draw
      const double part = uniform() * cdf[N - 1];
      cand[j] = static_cast<uint32_t>(std::min<size_t>(std::lower_bound(cdf.begin(), cdf.end(), part) - cdf.begin(), N - 1));
      rand_a[j] = static_cast<float>(uniform());
    }
    for (size_t i = 0; i < devs.size(); i++) {
      Dev& d = devs[i];
      sc[i].slots.clear();
      uint32_t cnt = 0;
      for (uint32_t j = 0; j < m; j++)
        if (cand[j] >= d.off && cand[j] < d.off + d.len) {
          local[cnt++] = cand[j] - d.off;
          sc[i].slots.push_back(j);
        }
      if (cnt == 0) continue;
      KMB_CU(cudaSetDevice(d.dev), kmcudaRuntimeError);
      KMB_CU(cudaMemcpyAsync(sc[i].rows.get(), local.data(), sizeof(uint32_t) * cnt, cudaMemcpyHostToDevice, d.st),
             kmcudaMemoryCopyError);
      KMB_CU(cudaStreamSynchronize(d.st), kmcudaRuntimeError);   // `local` is reused for the next shard
      KMB_CU(launch_afkmc2_min_dist(metric, d.X, d.C, D, k, sc[i].rows, cnt, sc[i].mind, d.st), kmcudaRuntimeError);
      KMB_CU(cudaMemcpyAsync(sc[i].host.data(), sc[i].mind.get(), sizeof(float) * cnt, cudaMemcpyDeviceToHost, d.st),
             kmcudaMemoryCopyError);
    }
    for (size_t i = 0; i < devs.size(); i++) {
      if (sc[i].slots.empty()) continue;
      KMB_CU(cudaSetDevice(devs[i].dev), kmcudaRuntimeError);
      KMB_CU(cudaStreamSynchronize(devs[i].st), kmcudaRuntimeError);
      for (size_t t = 0; t < sc[i].slots.size(); t++) {
        const float dmin = sc[i].host[t];
        const uint32_t slot = sc[i].slots[t];
        p_cand[slot] = weighted ? host_w[cand[slot]] * (dmin * dmin) : dmin * dmin;
      }
    }
    float curr_prob = 0;
    uint32_t curr_ind = 0;
    for (uint32_t j = 0; j < m; j++) {   // kmcuda.cc:382-389
      const float cand_prob = p_cand[j] / q[cand[j]];
      if (curr_prob == 0 || cand_prob / curr_prob > rand_a[j]) {
        curr_ind = j;
        curr_prob = cand_prob;
      }
    }
    float* dst = hostC.data() + static_cast<size_t>(k) * D;
    KMB_RET(fetch_row(cand[curr_ind], dst));
    for (auto& d : devs) {
      KMB_CU(cudaSetDevice(d.dev), kmcudaRuntimeError);
      KMB_CU(cudaMemcpyAsync(d.C.get() + static_cast<size_t>(k) * D, dst, sizeof(float) * D, cudaMemcpyHostToDevice, d.st),
             kmcudaMemoryCopyError);
    }
  }
  KMB_RET(sync_all());
  for (auto& d : devs) d.dists.release();
  return set_centroids_from_host(hostC.data());
}

// k-means|| (Bahmani et al., "Scalable K-Means++", VLDB 2012; DESIGN.md §4g).  c0 is k-means++'s first centroid; each
// of `rounds` rounds draws every row independently with probability l w_i d_i^2 / phi (l = 2K, d_i the true distance
// to the nearest candidate so far, phi = sum w_i d_i^2), runs one assignment pass against the round's new candidates
// only and lowers d_i where the winner is closer.  The candidates, weighted by the sample weight they are nearest to,
// are then clustered down to K by the library's own weighted k-means++ / Lloyd run; with at most K candidates they are
// the centroids and init_random's walk fills the rest.  Every shard draws its own rows with a counter hash of the
// global row index, so the draws do not depend on the device split.
KMCUDAResult Job::init_kmeans_parallel(uint32_t rounds, uint32_t seed) {
  std::vector<float> cand(D);          // the candidate rows in list order (round, row index), host copy
  std::vector<uint32_t> cand_rows(1);  // their global row indices
  KMB_RET(draw_first_centroid(cand.data(), &cand_rows[0]));
  struct Work {
    DevBuf<float> table, gathered;     // this round's candidates (all shards'), this shard's drawn rows
    DevBuf<uint32_t> nearest, idx, count;
    DevBuf<double> bsum, phi;
    DevBuf<uint8_t> flags;
    DevBuf<char> tmp;
    size_t tmp_bytes = 0;
    uint32_t nb = 0, drawn = 0;
  };
  std::vector<Work> wk(devs.size());
  for (size_t s = 0; s < devs.size(); s++) {
    Dev& d = devs[s];
    Work& w = wk[s];
    KMB_CU(cudaSetDevice(d.dev), kmcudaRuntimeError);
    w.nb = kmp_blocks(d.len);
    w.tmp_bytes = kmp_select_bytes(d.len);
    KMB_CU(d.dists.alloc(d.len), kmcudaMemoryAllocationFailure);
    KMB_CU(w.nearest.alloc(d.len), kmcudaMemoryAllocationFailure);
    KMB_CU(w.idx.alloc(d.len), kmcudaMemoryAllocationFailure);
    KMB_CU(w.count.alloc(1), kmcudaMemoryAllocationFailure);
    KMB_CU(w.bsum.alloc(w.nb), kmcudaMemoryAllocationFailure);
    KMB_CU(w.phi.alloc(1), kmcudaMemoryAllocationFailure);
    KMB_CU(w.flags.alloc(d.len), kmcudaMemoryAllocationFailure);
    KMB_CU(w.tmp.alloc(w.tmp_bytes), kmcudaMemoryAllocationFailure);
    KMB_CU(w.table.alloc(D), kmcudaMemoryAllocationFailure);
    KMB_CU(cudaMemcpyAsync(w.table.get(), cand.data(), sizeof(float) * D, cudaMemcpyHostToDevice, d.st),
           kmcudaMemoryCopyError);
    KMB_CU(launch_kmp_update(metric, d.X, d.len, D, w.table, 1, nullptr, 0, d.dists, w.nearest, d.w.get(), w.bsum, d.st),
           kmcudaRuntimeError);
    KMB_CU(launch_kmp_sum(w.bsum, w.nb, w.phi, d.st), kmcudaRuntimeError);
  }
  const double ell = 2.0 * K;
  for (uint32_t r = 1; r <= rounds; r++) {
    double phi = 0;
    for (auto& w : wk) w.drawn = 0;
    for (size_t s = 0; s < devs.size(); s++) {   // device order: the same total on every run
      double part = 0;
      KMB_CU(cudaSetDevice(devs[s].dev), kmcudaRuntimeError);
      KMB_CU(cudaMemcpyAsync(&part, wk[s].phi.get(), sizeof(double), cudaMemcpyDeviceToHost, devs[s].st),
             kmcudaMemoryCopyError);
      KMB_CU(cudaStreamSynchronize(devs[s].st), kmcudaRuntimeError);
      phi += part;
    }
    if (!(phi > 0)) break;   // every row sits on a candidate
    for (size_t s = 0; s < devs.size(); s++) {
      Dev& d = devs[s];
      Work& w = wk[s];
      KMB_CU(cudaSetDevice(d.dev), kmcudaRuntimeError);
      KMB_CU(launch_kmp_draw(d.dists, d.w.get(), d.len, d.off, seed, r, ell, phi, w.flags, w.idx, w.count, w.tmp,
                             w.tmp_bytes, d.st), kmcudaRuntimeError);
      KMB_CU(cudaMemcpyAsync(&w.drawn, w.count.get(), sizeof(uint32_t), cudaMemcpyDeviceToHost, d.st),
             kmcudaMemoryCopyError);
    }
    KMB_RET(sync_all());
    const uint32_t base = static_cast<uint32_t>(cand_rows.size());
    uint32_t fresh = 0;
    for (auto& w : wk) fresh += w.drawn;
    KMB_INFO("k-means|| round %" PRIu32 ": %" PRIu32 " candidates, cost %.17g\n", r, fresh, phi);
    if (fresh == 0) continue;   // nothing changes: the next round draws again from the same d
    // gather each shard's drawn rows, then every device gets the whole round's table in device (= row) order
    cand_rows.resize(base + fresh);
    for (size_t s = 0, at = base; s < devs.size(); s++) {
      Dev& d = devs[s];
      Work& w = wk[s];
      if (w.drawn == 0) continue;
      KMB_CU(cudaSetDevice(d.dev), kmcudaRuntimeError);
      KMB_CU(w.gathered.alloc(static_cast<size_t>(w.drawn) * D), kmcudaMemoryAllocationFailure);
      KMB_CU(launch_kmp_gather(d.X, D, w.idx, w.drawn, w.gathered, d.st), kmcudaRuntimeError);
      KMB_CU(cudaMemcpyAsync(cand_rows.data() + at, w.idx.get(), sizeof(uint32_t) * w.drawn, cudaMemcpyDeviceToHost,
                             d.st), kmcudaMemoryCopyError);
      at += w.drawn;
    }
    KMB_RET(sync_all());
    for (size_t s = 0, at = base; s < devs.size(); s++) {
      for (uint32_t j = 0; j < wk[s].drawn; j++) cand_rows[at + j] += devs[s].off;
      at += wk[s].drawn;
    }
    for (size_t t = 0; t < devs.size(); t++) {
      Dev& d = devs[t];
      KMB_CU(cudaSetDevice(d.dev), kmcudaRuntimeError);
      KMB_CU(wk[t].table.alloc(static_cast<size_t>(fresh) * D), kmcudaMemoryAllocationFailure);
      size_t at = 0;
      for (size_t s = 0; s < devs.size(); s++) {
        if (wk[s].drawn == 0) continue;
        KMB_CU(cudaMemcpyPeerAsync(wk[t].table.get() + at * D, d.dev, wk[s].gathered.get(), devs[s].dev,
                                   sizeof(float) * wk[s].drawn * D, d.st), kmcudaMemoryCopyError);
        at += wk[s].drawn;
      }
    }
    cand.resize(static_cast<size_t>(base + fresh) * D);
    KMB_CU(cudaSetDevice(devs[0].dev), kmcudaRuntimeError);
    KMB_CU(cudaMemcpyAsync(cand.data() + static_cast<size_t>(base) * D, wk[0].table.get(),
                           sizeof(float) * static_cast<size_t>(fresh) * D, cudaMemcpyDeviceToHost, devs[0].st),
           kmcudaMemoryCopyError);
    KMB_RET(sync_all());   // (the peer copies have read every `gathered` buffer)
    // one assignment pass of every shard against the round's candidates, then the running-minimum update
    std::vector<std::unique_ptr<Shard>> pass(devs.size());
    for (size_t s = 0; s < devs.size(); s++) {
      Dev& d = devs[s];
      Work& w = wk[s];
      pass[s].reset(new Shard(metric, d.dev, d.len, D, fresh, verbosity));
      KMB_RET(pass[s]->create(false));
      KMB_CU(cudaSetDevice(d.dev), kmcudaRuntimeError);
      KMB_CU(cudaMemsetAsync(d.assign.get(), 0xff, sizeof(uint32_t) * d.len, d.st), kmcudaRuntimeError);
      KMB_RET(pass[s]->assign(d.len, d.X, w.table, d.assign, d.prev, d.d_changed, d.st));
      KMB_CU(launch_kmp_update(metric, d.X, d.len, D, w.table, fresh, d.assign, base, d.dists, w.nearest, d.w.get(),
                               w.bsum, d.st), kmcudaRuntimeError);
      KMB_CU(launch_kmp_sum(w.bsum, w.nb, w.phi, d.st), kmcudaRuntimeError);
    }
    KMB_RET(sync_all());
    for (auto& p : pass) KMB_RET(p->check_pipeline());
  }
  const uint32_t Cn = static_cast<uint32_t>(cand_rows.size());
  KMB_INFO("k-means||: %" PRIu32 " candidates -> %" PRIu32 " centroids\n", Cn, K);
  g_prof.mark("init: k-means|| rounds");
  std::vector<float> hostC(static_cast<size_t>(K) * D);
  if (Cn <= K) {
    // the candidates, then init_random's walk from srand(seed) over the rows not chosen yet (and of positive weight)
    memcpy(hostC.data(), cand.data(), sizeof(float) * static_cast<size_t>(Cn) * D);
    std::vector<char> taken(N, 0);
    for (uint32_t i : cand_rows) taken[i] = 1;
    srand(seed);
    const std::vector<uint32_t> order = random_order(N);
    uint32_t c = Cn;
    for (uint32_t s = 0; s < N && c < K; s++) {
      const uint32_t i = order[s];
      if (taken[i] || (weighted && !(host_w[i] > 0.f))) continue;
      KMB_RET(fetch_row(i, hostC.data() + static_cast<size_t>(c) * D));
      c++;
    }
    if (c < K) {
      KMB_INFO("k-means||: only %" PRIu32 " samples have a positive weight, %" PRIu32 " clusters\n", c, K);
      return kmcudaInvalidArguments;
    }
    for (auto& d : devs) d.dists.release();
    KMB_RET(set_centroids_from_host(hostC.data()));
    g_prof.mark("init: k-means|| recluster");
    return kmcudaSuccess;
  }
  // candidate weights W_j = sum of w_i over the rows nearest to candidate j: exact counts, or compensated fp32 sums per
  // device added in device order (the weighted update's rule)
  std::vector<float> W(Cn, 0.f);
  {
    std::vector<uint32_t> total(Cn, 0), part_u(Cn);
    std::vector<float> part_f(Cn);
    for (size_t s = 0; s < devs.size(); s++) {
      Dev& d = devs[s];
      Work& w = wk[s];
      KMB_CU(cudaSetDevice(d.dev), kmcudaRuntimeError);
      if (weighted) {
        DevBuf<uint32_t> keys, start;
        DevBuf<float> wsorted, Wd;
        const size_t bytes = kmp_weights_bytes(d.len);
        KMB_CU(keys.alloc(d.len), kmcudaMemoryAllocationFailure);
        KMB_CU(start.alloc(2 * static_cast<size_t>(Cn)), kmcudaMemoryAllocationFailure);
        KMB_CU(wsorted.alloc(d.len), kmcudaMemoryAllocationFailure);
        KMB_CU(Wd.alloc(Cn), kmcudaMemoryAllocationFailure);
        KMB_CU(w.tmp.alloc(bytes), kmcudaMemoryAllocationFailure);
        KMB_CU(launch_kmp_weights(w.nearest, d.w, d.len, Cn, keys, wsorted, start, w.tmp, bytes, Wd, d.st),
               kmcudaRuntimeError);
        KMB_CU(cudaMemcpyAsync(part_f.data(), Wd.get(), sizeof(float) * Cn, cudaMemcpyDeviceToHost, d.st),
               kmcudaMemoryCopyError);
        KMB_CU(cudaStreamSynchronize(d.st), kmcudaRuntimeError);
        for (uint32_t j = 0; j < Cn; j++) W[j] += part_f[j];
      } else {
        DevBuf<uint32_t> counts;
        KMB_CU(counts.alloc(Cn), kmcudaMemoryAllocationFailure);
        KMB_CU(cudaMemsetAsync(counts.get(), 0, sizeof(uint32_t) * Cn, d.st), kmcudaRuntimeError);
        KMB_CU(launch_kmp_counts(w.nearest, d.len, counts, d.st), kmcudaRuntimeError);
        KMB_CU(cudaMemcpyAsync(part_u.data(), counts.get(), sizeof(uint32_t) * Cn, cudaMemcpyDeviceToHost, d.st),
               kmcudaMemoryCopyError);
        KMB_CU(cudaStreamSynchronize(d.st), kmcudaRuntimeError);
        for (uint32_t j = 0; j < Cn; j++) total[j] += part_u[j];
      }
    }
    if (!weighted)
      for (uint32_t j = 0; j < Cn; j++) W[j] = static_cast<float>(total[j]);
  }
  for (auto& d : devs) d.dists.release();
  wk.clear();
  // recluster: the steps of kmcuda_b200_kmeans_weighted(k-means++, tolerance 0.01, yinyang_t 0, metric, seed,
  // verbosity 0) on the candidate rows on the first device, with the same result.  Its phases stay out of the caller's
  // profile and log.  Two checks of the public call do not apply to the nested run:
  // - the unit-length probe of angular samples: the call's own samples passed it or were fp16x2, whose widened rows
  //   are unit length only to fp16 precision;
  // - KMCUDA_B200_STRICT_UPDATE=1, which replays the reference's unweighted update and would drop the weights W.
  {
    const bool prof = g_prof.on;
    g_prof.on = false;
    Job sub(metric, Cn, D, K, 0);
    sub.weighted = true;
    KMCUDAResult res = sub.setup({devs[0].dev}, true);
    if (res == kmcudaSuccess) {
      sub.devs[0].shard->strict_update = false;
      res = sub.ingest(cand.data(), W.data(), -1, false);
    }
    if (res == kmcudaSuccess) res = sub.check_weights();
    if (res == kmcudaSuccess) {
      srand(seed);
      res = sub.init_plusplus();
    }
    if (res == kmcudaSuccess) res = sub.yinyang(0.01f, 0);
    g_prof.on = prof;
    KMB_RET(res);
    KMB_CU(cudaSetDevice(devs[0].dev), kmcudaRuntimeError);
    KMB_CU(cudaMemcpy(hostC.data(), sub.devs[0].C.get(), sizeof(float) * hostC.size(), cudaMemcpyDeviceToHost),
           kmcudaMemoryCopyError);
  }
  KMB_RET(set_centroids_from_host(hostC.data()));
  g_prof.mark("init: k-means|| recluster");
  return kmcudaSuccess;
}

KMCUDAResult Job::init_centroids(KMCUDAInitMethod method, const void* init_params, uint32_t seed,
                                 int device_ptrs, bool fp16x2, const float* user_centroids) {
  if (metric == 1 && !fp16x2) {  // three probe samples must be unit length (kmcuda.cc:195-219)
    std::vector<float> row(D);
    for (uint32_t s : {0u, N / 2, N - 1}) {
      KMB_RET(fetch_row(s, row.data()));
      double norm = 0;
      for (int f = 0; f < D; f++) norm += row[f] * row[f];
      const float high = 1.00001, low = 0.99999;
      if (norm > high || norm < low) {
        KMB_INFO("error: angular distance: samples[%" PRIu32 "] has L2 norm = %f which is outside [%f, %f]\n",
                 s, norm, low, high);
        return kmcudaInvalidArguments;
      }
    }
  }
  srand(seed);
  switch (method) {
    case kmcudaInitMethodImport: {
      const size_t count = static_cast<size_t>(K) * D;
      for (auto& d : devs) {
        KMB_CU(cudaSetDevice(d.dev), kmcudaRuntimeError);
        if (!fp16x2) {
          if (device_ptrs < 0)
            KMB_CU(cudaMemcpyAsync(d.C.get(), user_centroids, count * 4, cudaMemcpyHostToDevice, d.st), kmcudaMemoryCopyError);
          else
            KMB_CU(cudaMemcpyPeerAsync(d.C.get(), d.dev, user_centroids, device_ptrs, count * 4, d.st), kmcudaMemoryCopyError);
        } else {
          DevBuf<char> tmp;
          KMB_CU(tmp.alloc(count * 2), kmcudaMemoryAllocationFailure);
          if (device_ptrs < 0)
            KMB_CU(cudaMemcpyAsync(tmp.get(), user_centroids, count * 2, cudaMemcpyHostToDevice, d.st), kmcudaMemoryCopyError);
          else
            KMB_CU(cudaMemcpyPeerAsync(tmp.get(), d.dev, user_centroids, device_ptrs, count * 2, d.st), kmcudaMemoryCopyError);
          KMB_CU(launch_half_to_float(tmp.get(), d.C.get(), count, d.st), kmcudaRuntimeError);
          KMB_CU(cudaStreamSynchronize(d.st), kmcudaMemoryCopyError);
        }
      }
      KMB_RET(sync_all());
      break;
    }
    case kmcudaInitMethodRandom:
      KMB_RET(init_random());
      break;
    case kmcudaInitMethodPlusPlus:
      KMB_RET(init_plusplus());
      break;
    case kmcudaInitMethodAFKMC2: {
      uint32_t m = init_params ? *reinterpret_cast<const uint32_t*>(init_params) : 0;
      if (m == 0) {
        m = 200;
      } else if (m > N / 2) {
        KMB_INFO("afkmc2: m > %" PRIu32 " is not supported (got %" PRIu32 ")\n", N / 2, m);
        return kmcudaInvalidArguments;
      }
      KMB_RET(init_afkmc2(m, seed));
      break;
    }
    case kmcudaInitMethodKMeansParallel: {
      const uint32_t r = init_params ? *reinterpret_cast<const uint32_t*>(init_params) : 0;
      KMB_RET(init_kmeans_parallel(r ? r : kKMeansParallelRounds, seed));   // (r <= 32: kmeans_impl)
      break;
    }
    default:
      return kmcudaInvalidArguments;
  }
  KMB_INFO("\rdone            \n");
  return kmcudaSuccess;
}

// one assignment pass over every shard; *changed = total reassignments
KMCUDAResult Job::assign_pass(uint32_t* changed) {
  for (auto& d : devs) {
    KMB_CU(cudaSetDevice(d.dev), kmcudaRuntimeError);
    KMB_CU(cudaMemsetAsync(d.d_changed.get(), 0, sizeof(uint32_t), d.st), kmcudaRuntimeError);
    KMB_RET(d.shard->assign(d.len, d.X, d.C, d.assign, d.prev, d.d_changed, d.st));
  }
  uint32_t total = 0;
  for (auto& d : devs) {
    uint32_t mine = 0;
    KMB_CU(cudaSetDevice(d.dev), kmcudaRuntimeError);
    KMB_CU(cudaMemcpyAsync(&mine, d.d_changed.get(), sizeof(mine), cudaMemcpyDeviceToHost, d.st), kmcudaMemoryCopyError);
    KMB_CU(cudaStreamSynchronize(d.st), kmcudaRuntimeError);
    total += mine;
    KMB_RET(d.shard->check_pipeline());
  }
  *changed = total;
  return kmcudaSuccess;
}

// centroid update: shard partial sums -> exchange (peer-memory reduce, or NCCL all-reduce) -> normalise on every GPU
KMCUDAResult Job::update() {
  if (devs.size() == 1 && devs[0].shard->strict_update) {
    // strict parity mode: the reference's running sums in sample order (bit-identical centroids, one GPU)
    Dev& d = devs[0];
    KMB_CU(cudaSetDevice(d.dev), kmcudaRuntimeError);
    return d.shard->update_reference_order(d.len, d.X, d.assign, d.prev, d.C, d.ccounts, d.st);
  }
  if (devs.size() > 1 && peer_exchange) {
    // nobody may overwrite its partial sums while a peer of the previous iteration is still reading them
    for (auto& d : devs) {
      KMB_CU(cudaSetDevice(d.dev), kmcudaRuntimeError);
      for (auto& e : devs)
        if (&e != &d) KMB_CU(cudaStreamWaitEvent(d.st, e.ev_reduced, 0), kmcudaRuntimeError);
    }
  }
  for (auto& d : devs) {
    KMB_CU(cudaSetDevice(d.dev), kmcudaRuntimeError);
    KMB_RET(d.shard->partial_sums(d.len, d.X, d.assign, d.sums, d.counts, d.st, d.w.get(), d.wsums.get()));
    if (devs.size() > 1 && peer_exchange) KMB_CU(cudaEventRecord(d.ev_partial, d.st), kmcudaRuntimeError);
  }
  if (devs.size() > 1 && peer_exchange) {
    PeerBuffers pb;
    PeerF32 pw;   // weighted: the per-cluster weight totals travel with the sums
    pb.n = pw.n = static_cast<int>(devs.size());
    for (size_t i = 0; i < devs.size(); i++) {
      pb.sums[i] = devs[i].sums.get();
      pb.counts[i] = devs[i].counts.get();
      pw.p[i] = devs[i].wsums.get();
    }
    for (auto& d : devs) {
      KMB_CU(cudaSetDevice(d.dev), kmcudaRuntimeError);
      for (auto& e : devs)
        if (&e != &d) KMB_CU(cudaStreamWaitEvent(d.st, e.ev_partial, 0), kmcudaRuntimeError);
      KMB_CU(launch_peer_reduce(pb, K, D, d.rsums, d.rcounts, d.st), kmcudaRuntimeError);
      if (weighted) KMB_CU(launch_peer_sum_f32(pw, K, d.rweights, d.st), kmcudaRuntimeError);
      KMB_CU(cudaEventRecord(d.ev_reduced, d.st), kmcudaRuntimeError);
      KMB_RET(d.shard->finish_update(d.rsums, d.rcounts, d.C, d.ccounts, d.st, d.rweights.get(), d.cweights.get()));
    }
    return kmcudaSuccess;
  }
  if (devs.size() > 1) {
    const NcclApi& nc = nccl_api();
    ncclResult_t r = nc.GroupStart();
    for (auto& d : devs) {
      if (r != ncclSuccess) break;
      r = nc.AllReduce(d.sums.get(), d.sums.get(), static_cast<size_t>(K) * D, ncclFloat32, ncclSum, d.comm, d.st);
      if (r == ncclSuccess)
        r = nc.AllReduce(d.counts.get(), d.counts.get(), K, ncclUint32, ncclSum, d.comm, d.st);
      if (r == ncclSuccess && weighted)
        r = nc.AllReduce(d.wsums.get(), d.wsums.get(), K, ncclFloat32, ncclSum, d.comm, d.st);
    }
    ncclResult_t rend = nc.GroupEnd();
    if (r == ncclSuccess) r = rend;
    if (r != ncclSuccess) {
      KMB_INFO("ncclAllReduce failed: %s\n", nc.GetErrorString(r));
      drop_cached_comms();   // a communicator that reported an error is not reused by later calls
      return kmcudaRuntimeError;
    }
  }
  for (auto& d : devs) {
    KMB_CU(cudaSetDevice(d.dev), kmcudaRuntimeError);
    KMB_RET(d.shard->finish_update(d.sums, d.counts, d.C, d.ccounts, d.st, d.wsums.get(), d.cweights.get()));
  }
  return kmcudaSuccess;
}

// reference kmeans_cuda_lloyd, kmeans.cu:934-1026 (resume == false)
KMCUDAResult Job::lloyd(float tolerance, int* iter_out, uint32_t* changed_out) {
  for (auto& d : devs) {
    KMB_CU(cudaSetDevice(d.dev), kmcudaRuntimeError);
    KMB_CU(cudaMemsetAsync(d.ccounts.get(), 0, sizeof(uint32_t) * K, d.st), kmcudaRuntimeError);
    if (d.cweights.get()) KMB_CU(cudaMemsetAsync(d.cweights.get(), 0, sizeof(float) * K, d.st), kmcudaRuntimeError);
    KMB_RET(d.shard->reset_update_state(d.st));
    KMB_CU(cudaMemsetAsync(d.assign.get(), 0xff, sizeof(uint32_t) * d.len, d.st), kmcudaRuntimeError);
    KMB_CU(cudaMemsetAsync(d.prev.get(), 0xff, sizeof(uint32_t) * d.len, d.st), kmcudaRuntimeError);
  }
  auto t_prev = std::chrono::steady_clock::now();
  for (int iter = 1;; iter++) {
    uint32_t changed = 0;
    KMB_RET(assign_pass(&changed));
    g_prof.mark("assign pass");
    // iteration period (update of the previous iteration + this pass; assign_pass synchronises): what a Yinyang
    // iteration has to beat (Job::yinyang)
    const auto t_now = std::chrono::steady_clock::now();
    if (iter >= 2) {
      const double ms = std::chrono::duration<double, std::milli>(t_now - t_prev).count();
      if (lloyd_iter_ms == 0 || ms < lloyd_iter_ms) lloyd_iter_ms = ms;
    }
    t_prev = t_now;
    KMB_INFO("iteration %d: %" PRIu32 " reassignments\n", iter, changed);
    if (iter_out) *iter_out = iter;
    if (changed_out) *changed_out = changed;
    if (changed <= tolerance * N) return kmcudaSuccess;  // float compare, kmeans.cu:707
    KMB_RET(update());
    g_prof.mark("centroid update");
  }
}

// Lloyd iterations from the current state (assignments belong to the current centroids, the update is due): used when
// the Yinyang iterations of a run turn out slower than its Lloyd passes (Job::yinyang)
KMCUDAResult Job::lloyd_continue(float tolerance, int iter) {
  for (;;) {
    KMB_RET(update());
    g_prof.mark("centroid update");
    iter++;
    uint32_t changed = 0;
    KMB_RET(assign_pass(&changed));
    g_prof.mark("assign pass");
    KMB_INFO("iteration %d: %" PRIu32 " reassignments\n", iter, changed);
    if (changed <= tolerance * N) return kmcudaSuccess;
  }
}

// Yinyang groups = k-means (k-means++ with srand(0), Lloyd to 2 %) over the K centroids,
// reference kmeans.cu:1061-1094.  Runs on the first device, result broadcast by the caller.
KMCUDAResult Job::group_centroids(uint32_t G, std::vector<uint32_t>* groups) {
  Job sub(metric, K, D, G, verbosity);
  std::vector<int> one{devs[0].dev};
  KMB_RET(sub.setup(one, false));
  sub.devs[0].X.borrow(devs[0].C.get());
  srand(0);
  KMB_RET(sub.init_plusplus());
  KMB_INFO("\rdone            \n");
  KMB_RET(sub.lloyd(kYinyangGroupTolerance, nullptr, nullptr));
  groups->resize(K);
  KMB_CU(cudaSetDevice(devs[0].dev), kmcudaRuntimeError);
  KMB_CU(cudaMemcpy(groups->data(), sub.devs[0].assign.get(), sizeof(uint32_t) * K, cudaMemcpyDeviceToHost),
         kmcudaMemoryCopyError);
  // The grouping only steers how tight the bounds are, never the result.  The exact part of a bounds refresh costs
  // |group(a_i)| distances per sample, so a degenerate grouping (near-equidistant centroids: one group swallows most
  // of them) is evened out: centroids in (group, index) order are cut into G runs of equal length.
  {
    std::vector<uint32_t> gsz(G, 0);
    uint32_t live = 0;
    for (uint32_t c = 0; c < K; c++)
      if ((*groups)[c] < G) { gsz[(*groups)[c]]++; live++; }
    const uint32_t avg = (live + G - 1) / G, biggest = *std::max_element(gsz.begin(), gsz.end());
    if (avg && biggest > 4 * avg) {
      KMB_INFO("Yinyang groups are unbalanced (largest %" PRIu32 ", average %" PRIu32 "): evened out\n", biggest, avg);
      std::vector<uint32_t> order;
      order.reserve(live);
      for (uint32_t c = 0; c < K; c++)
        if ((*groups)[c] < G) order.push_back(c);
      std::stable_sort(order.begin(), order.end(), [&](uint32_t x, uint32_t y) { return (*groups)[x] < (*groups)[y]; });
      for (uint32_t i = 0; i < live; i++) (*groups)[order[i]] = static_cast<uint32_t>(static_cast<uint64_t>(i) * G / live);
    }
  }
  return kmcudaSuccess;
}

// reference kmeans_cuda_yy, kmeans.cu:1028-1263
KMCUDAResult Job::yinyang(float tolerance, uint32_t G) {
  if (G == 0 || kYinyangDraftReassignments <= tolerance) {
    if (verbosity > 0) {
      if (G == 0) printf("too few clusters for this yinyang_t => Lloyd\n");
      else printf("tolerance is too high (>= %.2f) => Lloyd\n", kYinyangDraftReassignments);
    }
    return lloyd(tolerance, nullptr, nullptr);
  }
  KMB_INFO("running Lloyd until reassignments drop below %" PRIu32 "\n",
           static_cast<uint32_t>(kYinyangDraftReassignments * N));
  int iter = 0;
  uint32_t changed = 0;
  KMB_RET(lloyd(kYinyangDraftReassignments, &iter, &changed));
  if (changed <= tolerance * N) return kmcudaSuccess;
  std::vector<uint32_t> groups;
  KMB_RET(group_centroids(G, &groups));
  g_prof.mark("yinyang: group centroids");
  for (auto& d : devs) {
    KMB_RET(d.shard->enable_yinyang(G));
    KMB_CU(cudaSetDevice(d.dev), kmcudaRuntimeError);
    KMB_CU(cudaMemcpyAsync(d.shard->groups.get(), groups.data(), sizeof(uint32_t) * K, cudaMemcpyHostToDevice, d.st),
           kmcudaMemoryCopyError);
    KMB_CU(cudaMemsetAsync(d.d_changed.get(), 0, sizeof(uint32_t), d.st), kmcudaRuntimeError);
    KMB_RET(d.shard->yy_prepare(groups.data(), d.st));
  }
  KMB_RET(sync_all());
  bool refresh = true;
  // A Yinyang iteration only pays when it beats a Lloyd pass of the same run, and with the tensor-core pass that takes a
  // large K (the bounds stream is 8 (G + 1) bytes per sample, the pass 2 K D flop).  Both are timed: once a clean Yinyang
  // iteration (no refresh in it) was slower than the fastest Lloyd iteration, the run continues with Lloyd passes --
  // the assignments are the same either way (KMCUDA_B200_YY_ADAPTIVE=0 keeps Yinyang).
  const char* ad = getenv("KMCUDA_B200_YY_ADAPTIVE");
  const bool adaptive = !(ad && ad[0] == '0') && lloyd_iter_ms > 0;
  auto t_prev = std::chrono::steady_clock::now();
  bool clean = false;          // the iteration that just ended contained no refresh
  for (;; iter++) {
    if (!refresh) {
      uint32_t total_changed = 0, total_passed = 0;
      for (auto& d : devs) {
        uint32_t c = 0, p = 0;
        KMB_CU(cudaSetDevice(d.dev), kmcudaRuntimeError);
        KMB_CU(cudaMemcpyAsync(&c, d.d_changed.get(), 4, cudaMemcpyDeviceToHost, d.st), kmcudaMemoryCopyError);
        KMB_CU(cudaMemcpyAsync(&p, d.shard->yy_counters.get() + 1, 4, cudaMemcpyDeviceToHost, d.st), kmcudaMemoryCopyError);
        KMB_CU(cudaStreamSynchronize(d.st), kmcudaRuntimeError);
        KMB_RET(d.shard->check_pipeline());
        total_changed += c;
        total_passed += p;
      }
      KMB_INFO("iteration %d: %" PRIu32 " reassignments\n", iter, total_changed);
      if (total_changed <= tolerance * N) return kmcudaSuccess;
      {
        const auto t_now = std::chrono::steady_clock::now();
        const double ms = std::chrono::duration<double, std::milli>(t_now - t_prev).count();
        t_prev = t_now;
        if (adaptive && clean && ms > lloyd_iter_ms) {
          KMB_INFO("a Yinyang iteration takes %.2f ms, a Lloyd iteration %.2f ms => Lloyd\n", ms, lloyd_iter_ms);
          return lloyd_continue(tolerance, iter);
        }
        clean = true;
      }
      for (auto& d : devs) {
        KMB_CU(cudaSetDevice(d.dev), kmcudaRuntimeError);
        KMB_CU(cudaMemsetAsync(d.d_changed.get(), 0, sizeof(uint32_t), d.st), kmcudaRuntimeError);
      }
      KMB_DEBUG("passed number: %" PRIu32 "\n", total_passed);
      if (1.f - (total_passed + 0.f) / N < kYinyangRefreshEpsilon) refresh = true;
    }
    if (refresh) {
      KMB_INFO("refreshing Yinyang bounds...\n");
      for (auto& d : devs) {
        KMB_CU(cudaSetDevice(d.dev), kmcudaRuntimeError);
        KMB_RET(d.shard->yy_refresh(d.len, d.X, d.C, d.assign, d.st));
      }
      refresh = false;
      clean = false;
      g_prof.mark("yinyang: bounds refresh");
    }
    for (auto& d : devs) {
      KMB_CU(cudaSetDevice(d.dev), kmcudaRuntimeError);
      KMB_CU(cudaMemcpyAsync(d.shard->oldC.get(), d.C.get(), sizeof(float) * static_cast<size_t>(K) * D,
                             cudaMemcpyDeviceToDevice, d.st), kmcudaMemoryCopyError);
    }
    KMB_RET(update());
    g_prof.mark("centroid update");
    for (auto& d : devs) {
      KMB_CU(cudaSetDevice(d.dev), kmcudaRuntimeError);
      KMB_RET(d.shard->yy_step(d.len, d.X, d.C, d.assign, d.prev, d.d_changed, d.st));
    }
    g_prof.mark("yinyang: filter + local step");
    if (g_prof.on) {   // marks synchronise, so the pinned counters of the last pass are valid
      Shard* s0 = devs[0].shard.get();
      uint32_t yc[4] = {0, 0, 0, 0}, rq = 0, ov = 0;
      cudaSetDevice(devs[0].dev);
      cudaMemcpy(yc, s0->yy_counters.get(), sizeof(yc), cudaMemcpyDeviceToHost);
      if (s0->tc) tc_last_stats(s0->tc, &rq, &ov);
      fprintf(stderr, "[kmcuda_b200 timing]   yy step (dev 0): tightened %u, passed %u, candidate rows %u, pairs %u, "
              "reference-order scan rows %u\n", yc[0], yc[1], rq, s0->tc ? tc_last_pairs(s0->tc) : 0u, ov);
    }
  }
}

// Mini-batch k-means (DESIGN.md §4h): scikit-learn's MiniBatchKMeans steps with this library's draws, on one GPU.  Each
// step draws b rows with replacement, assigns them exactly, blends the batch's weighted member sums into the centroids
// with the running weight totals W, and on the steps scikit-learn's rule picks turns the centroids of low W into batch
// rows.  The only host round trip of a step is the stop decision (batch inertia, sum of squared centroid moves, count of
// W == 0).  After the last step one ordinary assignment pass gives the assignments.
KMCUDAResult Job::minibatch(uint32_t batch_size, uint64_t max_steps, float tolerance, uint32_t seed) {
  static const double kReassignmentRatio = 0.01;
  static const int kMaxNoImprovement = 10;
  Dev& d = devs[0];
  KMB_CU(cudaSetDevice(d.dev), kmcudaRuntimeError);
  const uint32_t b = std::min(batch_size, N);
  const uint64_t steps = max_steps ? max_steps : 100ull * N / b;
  Shard bs(metric, d.dev, b, D, K, verbosity);
  KMB_RET(bs.create(true));
  const size_t kd = static_cast<size_t>(K) * D;
  DevBuf<float> Cn, S, Wb;
  DevBuf<uint32_t> rows, result, row_result, keys, counts, cidx_in, cidx, pos_in, picked, small;
  DevBuf<double> W, Wn, bsum, stats, dsq, wsorted, ekey_in, ekey, minkept;
  DevBuf<char> tmp;
  const uint32_t nb = mb_blocks(b);
  const size_t tmp_bytes = mb_reassign_bytes(b, K);
  KMB_CU(Cn.alloc(kd), kmcudaMemoryAllocationFailure);
  KMB_CU(S.alloc(kd), kmcudaMemoryAllocationFailure);
  KMB_CU(Wb.alloc(K), kmcudaMemoryAllocationFailure);
  KMB_CU(rows.alloc(b), kmcudaMemoryAllocationFailure);
  KMB_CU(result.alloc(b), kmcudaMemoryAllocationFailure);
  KMB_CU(row_result.alloc(N), kmcudaMemoryAllocationFailure);
  KMB_CU(keys.alloc(b), kmcudaMemoryAllocationFailure);
  KMB_CU(counts.alloc(K), kmcudaMemoryAllocationFailure);
  KMB_CU(cidx_in.alloc(K), kmcudaMemoryAllocationFailure);
  KMB_CU(cidx.alloc(K), kmcudaMemoryAllocationFailure);
  KMB_CU(pos_in.alloc(b), kmcudaMemoryAllocationFailure);
  KMB_CU(picked.alloc(b), kmcudaMemoryAllocationFailure);
  KMB_CU(small.alloc(2), kmcudaMemoryAllocationFailure);
  KMB_CU(W.alloc(K), kmcudaMemoryAllocationFailure);
  KMB_CU(Wn.alloc(K), kmcudaMemoryAllocationFailure);
  KMB_CU(bsum.alloc(nb), kmcudaMemoryAllocationFailure);
  KMB_CU(stats.alloc(3), kmcudaMemoryAllocationFailure);
  KMB_CU(dsq.alloc(K), kmcudaMemoryAllocationFailure);
  KMB_CU(wsorted.alloc(K), kmcudaMemoryAllocationFailure);
  KMB_CU(ekey_in.alloc(b), kmcudaMemoryAllocationFailure);
  KMB_CU(ekey.alloc(b), kmcudaMemoryAllocationFailure);
  KMB_CU(minkept.alloc(1), kmcudaMemoryAllocationFailure);
  KMB_CU(tmp.alloc(tmp_bytes), kmcudaMemoryAllocationFailure);
  KMB_CU(cudaMemsetAsync(W.get(), 0, sizeof(double) * K, d.st), kmcudaRuntimeError);
  // scikit-learn's _tolerance: tolerance times the mean of the unweighted per-feature variances
  double tol_abs = 0;
  if (tolerance > 0) {
    DevBuf<double> work, var;
    KMB_CU(work.alloc(mb_variance_doubles(D)), kmcudaMemoryAllocationFailure);
    KMB_CU(var.alloc(D), kmcudaMemoryAllocationFailure);
    KMB_CU(launch_mb_variance(d.X, N, D, work, var, d.st), kmcudaRuntimeError);
    std::vector<double> hv(D);
    KMB_CU(cudaMemcpyAsync(hv.data(), var.get(), sizeof(double) * D, cudaMemcpyDeviceToHost, d.st),
           kmcudaMemoryCopyError);
    KMB_CU(cudaStreamSynchronize(d.st), kmcudaRuntimeError);
    double m = 0;
    for (int f = 0; f < D; f++) m += hv[f];
    tol_abs = m / D * static_cast<double>(tolerance);
  }
  g_prof.mark("mini-batch: setup");
  MbReassign ra;
  ra.K = K;
  ra.b = b;
  ra.D = D;
  ra.ratio = kReassignmentRatio;
  ra.w = d.w.get();
  ra.X = d.X;
  ra.rows = rows;
  ra.cidx_in = cidx_in;
  ra.cidx = cidx;
  ra.pos_in = pos_in;
  ra.picked = picked;
  ra.npos = small.get();
  ra.m = small.get() + 1;
  ra.wsorted = wsorted;
  ra.ekey_in = ekey_in;
  ra.ekey = ekey;
  ra.minkept = minkept;
  ra.tmp = tmp.get();
  ra.tmp_bytes = tmp_bytes;
  float *cur = d.C.get(), *nxt = Cn.get();
  double *wcur = W.get(), *wnxt = Wn.get();
  const double alpha = std::min(1.0, 2.0 * b / (static_cast<double>(N) + 1));
  double ewa = 0, ewa_min = 0, h[3] = {0, 0, static_cast<double>(K)};
  bool have_ewa = false, have_min = false;
  int no_improvement = 0;
  uint64_t since_reassign = 0, s = 1;
  for (; s <= steps; s++) {
    // scikit-learn's _random_reassign, on the weight totals before this step
    since_reassign += b;
    const bool reassign = h[2] > 0 || since_reassign >= 10ull * K;
    if (reassign) since_reassign = 0;
    KMB_CU(launch_mb_draw(N, b, mb_step_key(seed, s, kMbTagBatch), rows, d.st), kmcudaRuntimeError);
    KMB_RET(bs.assign_rows(b, d.X, N, rows, cur, row_result, result, d.st));
    KMB_CU(launch_mb_inertia(d.X, rows, b, D, cur, K, result, d.w.get(), keys, bsum, d.st), kmcudaRuntimeError);
    KMB_CU(launch_kmp_sum(bsum, nb, stats.get(), d.st), kmcudaRuntimeError);
    // unweighted: the member counts are the weight totals (a weight of 1 per entry; all-ones weights give the same bits)
    KMB_RET(bs.partial_sums_rows(b, d.X, rows, keys, S, counts, d.st, d.w.get(), weighted ? Wb.get() : nullptr));
    KMB_CU(launch_mb_blend(cur, wcur, S, weighted ? Wb.get() : nullptr, counts, K, D, nxt, wnxt, d.st),
           kmcudaRuntimeError);
    if (reassign) {
      ra.key = mb_step_key(seed, s, kMbTagReassign);
      ra.C = nxt;
      ra.W = wnxt;
      KMB_CU(launch_mb_reassign(ra, d.st), kmcudaRuntimeError);
    }
    KMB_CU(launch_mb_stats(cur, nxt, wnxt, K, D, dsq, stats.get() + 1, d.st), kmcudaRuntimeError);
    KMB_CU(cudaMemcpyAsync(h, stats.get(), sizeof(h), cudaMemcpyDeviceToHost, d.st), kmcudaMemoryCopyError);
    KMB_CU(cudaStreamSynchronize(d.st), kmcudaRuntimeError);
    KMB_RET(bs.check_pipeline());
    std::swap(cur, nxt);
    std::swap(wcur, wnxt);
    // scikit-learn's _mini_batch_convergence
    const double mean = h[0] / b;
    if (s == 1) {
      KMB_INFO("mini-batch step %" PRIu64 "/%" PRIu64 ": mean batch inertia %.17g\n", s, steps, mean);
      continue;
    }
    ewa = have_ewa ? ewa * (1 - alpha) + mean * alpha : mean;
    have_ewa = true;
    KMB_INFO("mini-batch step %" PRIu64 "/%" PRIu64 ": mean batch inertia %.17g, ewa inertia %.17g\n", s, steps, mean,
             ewa);
    if (tol_abs > 0 && h[1] <= tol_abs) {
      KMB_INFO("mini-batch: converged (small centers change) at step %" PRIu64 "/%" PRIu64 "\n", s, steps);
      break;
    }
    if (!have_min || ewa < ewa_min) {
      no_improvement = 0;
      ewa_min = ewa;
      have_min = true;
    } else {
      no_improvement++;
    }
    if (no_improvement >= kMaxNoImprovement) {
      KMB_INFO("mini-batch: converged (lack of improvement in inertia) at step %" PRIu64 "/%" PRIu64 "\n", s, steps);
      break;
    }
  }
  if (s > steps) KMB_INFO("mini-batch: %" PRIu64 " steps\n", steps);
  if (cur != d.C.get())
    KMB_CU(cudaMemcpyAsync(d.C.get(), cur, sizeof(float) * kd, cudaMemcpyDeviceToDevice, d.st), kmcudaMemoryCopyError);
  g_prof.mark("mini-batch: steps");
  KMB_CU(cudaMemsetAsync(d.assign.get(), 0xff, sizeof(uint32_t) * d.len, d.st), kmcudaRuntimeError);
  KMB_CU(cudaMemsetAsync(d.prev.get(), 0xff, sizeof(uint32_t) * d.len, d.st), kmcudaRuntimeError);
  uint32_t changed = 0;
  KMB_RET(assign_pass(&changed));
  g_prof.mark("assign pass");
  return kmcudaSuccess;
}

KMCUDAResult Job::average_distance(float* out) {
  KMB_INFO("calculating the average distance...\n");
  double sum = 0;
  for (auto& d : devs) {
    KMB_CU(cudaSetDevice(d.dev), kmcudaRuntimeError);
    KMB_CU(cudaMemsetAsync(d.d_dsum.get(), 0, sizeof(double), d.st), kmcudaRuntimeError);
    KMB_CU(launch_average_distance(metric, d.X, d.C, d.len, D, d.assign, d.d_dsum, d.st, d.w.get()), kmcudaRuntimeError);
  }
  for (auto& d : devs) {
    double part = 0;
    KMB_CU(cudaSetDevice(d.dev), kmcudaRuntimeError);
    KMB_CU(cudaMemcpyAsync(&part, d.d_dsum.get(), sizeof(double), cudaMemcpyDeviceToHost, d.st), kmcudaMemoryCopyError);
    KMB_CU(cudaStreamSynchronize(d.st), kmcudaRuntimeError);
    sum += part;
  }
  *out = static_cast<float>(sum / (weighted ? wtotal : N));   // weighted: sum w d / sum w
  return kmcudaSuccess;
}

static KMCUDAResult print_memory_stats(const std::vector<int>& devs) {
  for (int dev : devs) {
    cudaSetDevice(dev);
    size_t free_bytes, total_bytes;
    if (cudaMemGetInfo(&free_bytes, &total_bytes) != cudaSuccess) return kmcudaRuntimeError;
    printf("GPU #%d memory: used %zu bytes (%.1f%%), free %zu bytes, total %zu bytes\n", dev,
           total_bytes - free_bytes, (total_bytes - free_bytes) * 100.0 / total_bytes, free_bytes, total_bytes);
  }
  return kmcudaSuccess;
}

}  // namespace kmb

using namespace kmb;

// kmeans_cuda and kmcuda_b200_kmeans_weighted (weights == nullptr: the unweighted run)
static KMCUDAResult kmeans_impl(KMCUDAInitMethod init, const void* init_params, float tolerance,
                                float yinyang_t, KMCUDADistanceMetric metric, uint32_t samples_size,
                                uint16_t features_size, uint32_t clusters_size, uint32_t seed,
                                uint32_t device, int32_t device_ptrs, int32_t fp16x2, int32_t verbosity,
                                const float* samples, const float* weights, float* centroids,
                                uint32_t* assignments, float* average_distance, bool minibatch = false,
                                uint32_t batch_size = 0, uint32_t max_steps = 0) {
  KMB_DEBUG("arguments: %d %p %.3f %.2f %d %" PRIu32 " %" PRIu16 " %" PRIu32 " %" PRIu32 " %" PRIu32
            " %d %" PRIi32 " %p %p %p %p\n", init, init_params, tolerance, yinyang_t, metric, samples_size,
            features_size, clusters_size, seed, device, fp16x2, verbosity, samples, centroids, assignments,
            average_distance);
  // argument validation: reference check_kmeans_args, kmcuda.cc:19-61
  if (clusters_size < 2 || clusters_size == UINT32_MAX) return kmcudaInvalidArguments;
  if (features_size == 0) return kmcudaInvalidArguments;
  if (samples_size < clusters_size) return kmcudaInvalidArguments;
  {
    int count = 0;
    cudaGetDeviceCount(&count);
    if (count < 32 && device > (1u << count)) return kmcudaNoSuchDevice;
  }
  if (samples == nullptr || centroids == nullptr || assignments == nullptr) return kmcudaInvalidArguments;
  if (!(tolerance >= 0 && tolerance <= 1)) return kmcudaInvalidArguments;
  if (!(yinyang_t >= 0 && yinyang_t <= 0.5)) return kmcudaInvalidArguments;
  if (static_cast<uint64_t>(features_size) * (fp16x2 ? 2 : 1) > 65535u) return kmcudaInvalidArguments;
  if (init == kmcudaInitMethodKMeansParallel && init_params &&
      *static_cast<const uint32_t*>(init_params) > kKMeansParallelMaxRounds)
    return kmcudaInvalidArguments;
  if (minibatch) {
    // one GPU, L2, a real batch; strict mode replays a Lloyd update that mini-batch steps do not have
    const char* su = getenv("KMCUDA_B200_STRICT_UPDATE");
    if (batch_size == 0 || metric == kmcudaDistanceMetricCosine || (device & (device - 1)) != 0 ||
        (su && su[0] == '1')) {
      KMB_INFO("mini-batch k-means takes batch_size >= 1, the L2 metric, one device and no strict update mode\n");
      return kmcudaInvalidArguments;
    }
    if (device == 0) device = 1;
  }
  if (weights) {
    // strict mode replays the reference's unweighted running sums; there is no weighted reference to replay
    const char* su = getenv("KMCUDA_B200_STRICT_UPDATE");
    if (su && su[0] == '1') {
      KMB_INFO("sample weights cannot be combined with KMCUDA_B200_STRICT_UPDATE=1\n");
      return kmcudaInvalidArguments;
    }
  }
  KMB_INFO("reassignments threshold: %" PRIu32 "\n", static_cast<uint32_t>(tolerance * samples_size));
  const uint32_t yy_groups_size = static_cast<uint32_t>(yinyang_t * clusters_size);
  KMB_DEBUG("yinyang groups: %" PRIu32 "\n", yy_groups_size);
  std::vector<int> dev_ids;
  KMB_RET(list_devices(device, verbosity, &dev_ids));
  enable_p2p(dev_ids, device_ptrs, verbosity);
  const int m = metric == kmcudaDistanceMetricCosine ? 1 : 0;
  const int D = static_cast<int>(features_size) * (fp16x2 ? 2 : 1);
  g_prof.begin(dev_ids);
  Job job(m, samples_size, D, clusters_size, verbosity);
  job.weighted = weights != nullptr;
  KMB_RET(job.setup(dev_ids, true));
  g_prof.mark("setup: exchange (peer / nccl)");
  KMB_RET(job.ingest(samples, weights, device_ptrs, fp16x2 != 0));
  g_prof.mark("ingest (H2D / peer copy)");
  if (weights) {
    KMB_RET(job.check_weights());
    g_prof.mark("weight check");
  }
  if (verbosity > 1) KMB_RET(print_memory_stats(dev_ids));
  KMB_RET(job.init_centroids(init, init_params, seed, device_ptrs, fp16x2 != 0, centroids));
  g_prof.mark("init centroids");
  if (minibatch) KMB_RET(job.minibatch(batch_size, max_steps, tolerance, seed));
  else KMB_RET(job.yinyang(tolerance, yy_groups_size));
  if (average_distance) KMB_RET(job.average_distance(average_distance));
  g_prof.mark("average distance");
  // copy-out: centroids from the first device (identical everywhere), assignment slices from each shard
  const size_t ccount = static_cast<size_t>(clusters_size) * D;
  {
    Dev& d0 = job.devs[0];
    KMB_CU(cudaSetDevice(d0.dev), kmcudaRuntimeError);
    const void* csrc = d0.C.get();
    DevBuf<char> tmp;
    if (fp16x2) {
      KMB_CU(tmp.alloc(ccount * 2), kmcudaMemoryAllocationFailure);
      KMB_CU(launch_float_to_half(d0.C.get(), tmp.get(), ccount, d0.st), kmcudaRuntimeError);
      csrc = tmp.get();
    }
    const size_t cbytes = ccount * (fp16x2 ? 2 : 4);
    if (device_ptrs < 0)
      KMB_CU(cudaMemcpyAsync(centroids, csrc, cbytes, cudaMemcpyDeviceToHost, d0.st), kmcudaMemoryCopyError);
    else
      KMB_CU(cudaMemcpyPeerAsync(centroids, device_ptrs, csrc, d0.dev, cbytes, d0.st), kmcudaMemoryCopyError);
    KMB_CU(cudaStreamSynchronize(d0.st), kmcudaMemoryCopyError);
  }
  for (auto& d : job.devs) {
    KMB_CU(cudaSetDevice(d.dev), kmcudaRuntimeError);
    if (device_ptrs < 0)
      KMB_CU(cudaMemcpyAsync(assignments + d.off, d.assign.get(), sizeof(uint32_t) * d.len,
                             cudaMemcpyDeviceToHost, d.st), kmcudaMemoryCopyError);
    else
      KMB_CU(cudaMemcpyPeerAsync(assignments + d.off, device_ptrs, d.assign.get(), d.dev,
                                 sizeof(uint32_t) * d.len, d.st), kmcudaMemoryCopyError);
  }
  KMB_RET(job.sync_all());
  g_prof.mark("copy-out");
  g_prof.report("kmeans_cuda");
  KMB_DEBUG("return kmcudaSuccess\n");
  return kmcudaSuccess;
}

extern "C" {

KMCUDAResult kmeans_cuda(KMCUDAInitMethod init, const void* init_params, float tolerance,
                         float yinyang_t, KMCUDADistanceMetric metric, uint32_t samples_size,
                         uint16_t features_size, uint32_t clusters_size, uint32_t seed,
                         uint32_t device, int32_t device_ptrs, int32_t fp16x2, int32_t verbosity,
                         const float* samples, float* centroids, uint32_t* assignments,
                         float* average_distance) {
  return kmeans_impl(init, init_params, tolerance, yinyang_t, metric, samples_size, features_size, clusters_size, seed,
                     device, device_ptrs, fp16x2, verbosity, samples, nullptr, centroids, assignments,
                     average_distance);
}

KMCUDAResult kmcuda_b200_kmeans_weighted(KMCUDAInitMethod init, const void* init_params, float tolerance,
                                         float yinyang_t, KMCUDADistanceMetric metric, uint32_t samples_size,
                                         uint16_t features_size, uint32_t clusters_size, uint32_t seed,
                                         uint32_t device, int32_t device_ptrs, int32_t fp16x2, int32_t verbosity,
                                         const float* samples, const float* weights, float* centroids,
                                         uint32_t* assignments, float* average_distance) {
  return kmeans_impl(init, init_params, tolerance, yinyang_t, metric, samples_size, features_size, clusters_size, seed,
                     device, device_ptrs, fp16x2, verbosity, samples, weights, centroids, assignments,
                     average_distance);
}

KMCUDAResult kmcuda_b200_kmeans_minibatch(KMCUDAInitMethod init, const void* init_params, float tolerance,
                                          KMCUDADistanceMetric metric, uint32_t samples_size,
                                          uint16_t features_size, uint32_t clusters_size, uint32_t seed,
                                          uint32_t device, int32_t device_ptrs, int32_t fp16x2, int32_t verbosity,
                                          const float* samples, const float* weights, uint32_t batch_size,
                                          uint32_t max_steps, float* centroids, uint32_t* assignments,
                                          float* average_distance) {
  return kmeans_impl(init, init_params, tolerance, 0.f, metric, samples_size, features_size, clusters_size, seed,
                     device, device_ptrs, fp16x2, verbosity, samples, weights, centroids, assignments,
                     average_distance, true, batch_size, max_steps);
}

KMCUDAResult knn_cuda(uint16_t k, KMCUDADistanceMetric metric, uint32_t samples_size,
                      uint16_t features_size, uint32_t clusters_size, uint32_t device,
                      int32_t device_ptrs, int32_t fp16x2, int32_t verbosity, const float* samples,
                      const float* centroids, const uint32_t* assignments, uint32_t* neighbors) {
  KMB_DEBUG("arguments: %" PRIu16 " %d %" PRIu32 " %" PRIu16 " %" PRIu32 " %" PRIu32 " %" PRIi32 " %" PRIi32
            " %" PRIi32 " %p %p %p %p\n", k, metric, samples_size, features_size, clusters_size, device,
            device_ptrs, fp16x2, verbosity, samples, centroids, assignments, neighbors);
  // reference check_knn_args, kmcuda.cc:537-570 (the reference computes but ignores the verdict,
  // kmcuda.cc:583-584; here invalid arguments are rejected)
  if (k == 0) return kmcudaInvalidArguments;
  if (clusters_size < 2 || clusters_size == UINT32_MAX) return kmcudaInvalidArguments;
  if (features_size == 0) return kmcudaInvalidArguments;
  if (samples_size < clusters_size) return kmcudaInvalidArguments;
  if (samples == nullptr || centroids == nullptr || assignments == nullptr || neighbors == nullptr)
    return kmcudaInvalidArguments;
  if (static_cast<uint64_t>(features_size) * (fp16x2 ? 2 : 1) > 65535u) return kmcudaInvalidArguments;
  std::vector<int> dev_ids;
  KMB_RET(list_devices(device, verbosity, &dev_ids));
  enable_p2p(dev_ids, device_ptrs, verbosity);
  const int m = metric == kmcudaDistanceMetricCosine ? 1 : 0;
  const int D = static_cast<int>(features_size) * (fp16x2 ? 2 : 1);
  const uint32_t N = samples_size, K = clusters_size;
  auto plan = split_rows(N, static_cast<uint32_t>(D) * sizeof(float), dev_ids.size());
  unsigned long long total_pairs = 0;
  g_prof.begin(dev_ids);
  struct KDev {
    DevBuf<float> X, C, cd, radii, heap;
    DevBuf<float> cd_l2, radii_l2;   // angular metric on the tensor-core route: its cluster pruning works in L2
    DevBuf<uint32_t> assign, inv_keys, iota, inv, off, counts, neigh;
    DevBuf<char> cub;
    DevBuf<unsigned long long> pairs;
    cudaStream_t st = nullptr;
    cudaEvent_t done = nullptr;
  };
  std::vector<std::unique_ptr<KDev>> kd;
  auto cleanup = [&]() {
    for (size_t i = 0; i < kd.size(); i++) {
      cudaSetDevice(dev_ids[i]);
      if (kd[i]->done) cudaEventDestroy(kd[i]->done);
      if (kd[i]->st) cudaStreamDestroy(kd[i]->st);
    }
  };
  // Several GPUs on the tensor-core path: every GPU holds all samples (as in the reference, kmcuda.cc:157-158) and
  // the cluster-aligned candidate table, and serves an equal share of the query TILES into its own full-size
  // neighbour array; device 0 merges the arrays over peer memory (element-wise minimum against the 0xFFFFFFFF fill).
  bool shard_tc = false;
  {
    const char* fx0 = getenv("KMCUDA_B200_FORCE_EXACT");
    shard_tc = dev_ids.size() > 1 && m == 0 && !(fx0 && fx0[0] == '1') && tc_knn_supported(m, k, N, D, K);
    for (size_t i = 0; i < dev_ids.size() && shard_tc; i++)
      for (size_t j = 0; j < dev_ids.size() && shard_tc; j++) {
        int access = 0;
        if (i != j && (cudaDeviceCanAccessPeer(&access, dev_ids[i], dev_ids[j]) != cudaSuccess || !access)) shard_tc = false;
      }
  }
  bool shard_tc_ok = shard_tc;
  // every device gets the whole sample matrix (candidates can live anywhere), its slice of queries.  With several
  // devices on the tensor-core path the per-device pipelines (which synchronise their own stream a few times) run
  // on one host thread each, so the GPUs work concurrently.
  for (size_t i = 0; i < dev_ids.size(); i++) kd.emplace_back(new KDev);
  std::atomic<bool> any_tc_miss{false};
  auto per_device = [&](size_t i) -> KMCUDAResult {
    KDev& d = *kd[i];
    const int dev = dev_ids[i];
    const uint32_t qlen = shard_tc ? N : plan[i].second;   // rows of this device's neighbour array
#define KNN_CU(call, code) do { cudaError_t e__ = (call); if (e__ != cudaSuccess) { KMB_INFO("%s:%d -> %s\n", __FILE__, __LINE__, cudaGetErrorString(e__)); return code; } } while (false)
    KNN_CU(cudaSetDevice(dev), kmcudaNoSuchDevice);
    KNN_CU(cudaStreamCreateWithFlags(&d.st, cudaStreamNonBlocking), kmcudaRuntimeError);
    KNN_CU(cudaEventCreateWithFlags(&d.done, cudaEventDisableTiming), kmcudaRuntimeError);
    const size_t xcount = static_cast<size_t>(N) * D, ccount = static_cast<size_t>(K) * D;
    auto load = [&](DevBuf<float>& dst, const float* src, size_t count) -> cudaError_t {
      cudaError_t e;
      if (!fp16x2) {
        if (device_ptrs >= 0 && device_ptrs == dev) { dst.borrow(const_cast<float*>(src)); return cudaSuccess; }
        if ((e = dst.alloc(count)) != cudaSuccess) return e;
        if (device_ptrs < 0) return host_to_device(dst.get(), src, count * 4, dev, d.st);
        return cudaMemcpyPeerAsync(dst.get(), dev, src, device_ptrs, count * 4, d.st);
      }
      if ((e = dst.alloc(count)) != cudaSuccess) return e;
      DevBuf<char> tmp;
      const void* hsrc = src;
      if (!(device_ptrs >= 0 && device_ptrs == dev)) {
        if ((e = tmp.alloc(count * 2)) != cudaSuccess) return e;
        e = device_ptrs < 0 ? host_to_device(tmp.get(), src, count * 2, dev, d.st)
                            : cudaMemcpyPeerAsync(tmp.get(), dev, src, device_ptrs, count * 2, d.st);
        if (e != cudaSuccess) return e;
        hsrc = tmp.get();
      }
      if ((e = launch_half_to_float(hsrc, dst.get(), count, d.st)) != cudaSuccess) return e;
      return cudaStreamSynchronize(d.st);
    };
    KNN_CU(load(d.X, samples, xcount), kmcudaMemoryCopyError);
    KNN_CU(load(d.C, centroids, ccount), kmcudaMemoryCopyError);
    if (device_ptrs >= 0 && device_ptrs == dev) {
      d.assign.borrow(const_cast<uint32_t*>(assignments));
    } else {
      KNN_CU(d.assign.alloc(N), kmcudaMemoryAllocationFailure);
      if (device_ptrs < 0) KNN_CU(cudaMemcpyAsync(d.assign.get(), assignments, 4ull * N, cudaMemcpyHostToDevice, d.st), kmcudaMemoryCopyError);
      else KNN_CU(cudaMemcpyPeerAsync(d.assign.get(), dev, assignments, device_ptrs, 4ull * N, d.st), kmcudaMemoryCopyError);
    }
    KNN_CU(d.inv_keys.alloc(N), kmcudaMemoryAllocationFailure);
    KNN_CU(d.iota.alloc(N), kmcudaMemoryAllocationFailure);
    KNN_CU(d.inv.alloc(N), kmcudaMemoryAllocationFailure);
    KNN_CU(d.off.alloc(static_cast<size_t>(K) + 1), kmcudaMemoryAllocationFailure);
    KNN_CU(d.counts.alloc(K), kmcudaMemoryAllocationFailure);
    KNN_CU(d.cd.alloc(static_cast<size_t>(K) * K), kmcudaMemoryAllocationFailure);
    KNN_CU(d.radii.alloc(K), kmcudaMemoryAllocationFailure);
    KNN_CU(d.heap.alloc(static_cast<size_t>(qlen) * 2 * k), kmcudaMemoryAllocationFailure);
    KNN_CU(d.neigh.alloc(static_cast<size_t>(qlen) * k), kmcudaMemoryAllocationFailure);
    KNN_CU(d.pairs.alloc(1), kmcudaMemoryAllocationFailure);
    KNN_CU(cudaMemsetAsync(d.pairs.get(), 0, sizeof(unsigned long long), d.st), kmcudaRuntimeError);
    if (shard_tc) KNN_CU(cudaMemsetAsync(d.neigh.get(), 0xff, sizeof(uint32_t) * static_cast<size_t>(qlen) * k, d.st), kmcudaRuntimeError);
    // inverse assignments (reference: host std::sort of (assignment, index) tuples, kmcuda.cc:648-691):
    // stable device radix sort + binary-searched CSR offsets
    if (i == 0) KMB_INFO("initializing the inverse assignments...\n");
    UpdateWorkspace ws;
    ws.cub_tmp_bytes = update_cub_bytes(N);
    KNN_CU(d.cub.alloc(ws.cub_tmp_bytes), kmcudaMemoryAllocationFailure);
    ws.cub_tmp = d.cub.get();
    if (dev_ids.size() == 1) g_prof.mark("knn: alloc + ingest");
    KNN_CU(launch_knn_inverse(d.assign, N, K, d.iota, d.inv_keys, d.inv, d.off, d.counts, ws, d.st), kmcudaRuntimeError);
    KNN_CU(launch_knn_radii(m, d.X, d.C, N, D, K, d.assign, d.radii, d.st), kmcudaRuntimeError);
    KNN_CU(launch_knn_centroid_distances(m, d.C, K, D, d.cd, d.st), kmcudaRuntimeError);
    KNN_CU(launch_knn_radii_fix(d.off, K, d.radii, d.st), kmcudaRuntimeError);
    if (dev_ids.size() == 1) g_prof.mark("knn: inverse, radii, centroid distances");
    bool searched = false;
    const char* fx = getenv("KMCUDA_B200_FORCE_EXACT");
    if ((dev_ids.size() == 1 || shard_tc) && !(fx && fx[0] == '1') && tc_knn_supported(m, k, N, D, K)) {
      // tensor-core candidate search; the rows it cannot serve go through the reference-order search below
      uint32_t nv = 0, tc_err = 0;
      KNN_CU(cudaMemcpyAsync(&nv, d.off.get() + K, sizeof(nv), cudaMemcpyDeviceToHost, d.st), kmcudaMemoryCopyError);
      KNN_CU(cudaStreamSynchronize(d.st), kmcudaRuntimeError);
      DevBuf<uint32_t> fb_rows, d_nfb;
      KNN_CU(fb_rows.alloc(N), kmcudaMemoryAllocationFailure);
      KNN_CU(d_nfb.alloc(1), kmcudaMemoryAllocationFailure);
      KNN_CU(cudaMemsetAsync(d_nfb.get(), 0, sizeof(uint32_t), d.st), kmcudaRuntimeError);
      cudaError_t te = cudaSuccess;
      const float *tcd = d.cd, *tradii = d.radii;
      if (m == 1 && nv >= 4096) {
        KNN_CU(d.cd_l2.alloc(static_cast<size_t>(K) * K), kmcudaMemoryAllocationFailure);
        KNN_CU(d.radii_l2.alloc(K), kmcudaMemoryAllocationFailure);
        KNN_CU(launch_knn_radii(0, d.X, d.C, N, D, K, d.assign, d.radii_l2, d.st), kmcudaRuntimeError);
        KNN_CU(launch_knn_centroid_distances(0, d.C, K, D, d.cd_l2, d.st), kmcudaRuntimeError);
        KNN_CU(launch_knn_radii_fix(d.off, K, d.radii_l2, d.st), kmcudaRuntimeError);
        tcd = d.cd_l2;
        tradii = d.radii_l2;
      }
      if (nv >= 4096)
        te = tc_knn_search(m, k, d.X, d.C, N, D, K, d.assign, d.inv, d.off, tcd, tradii, nv, d.neigh, fb_rows, d_nfb,
                           d.pairs, &tc_err, shard_tc ? static_cast<uint32_t>(i) : 0u,
                           shard_tc ? static_cast<uint32_t>(dev_ids.size()) : 1u, d.st);
      if (dev_ids.size() == 1) g_prof.mark("knn: tensor-core candidate search");
      if (nv >= 4096 && te == cudaSuccess && tc_err == 0) {
        if (i == 0) KNN_CU(launch_knn_tail_rows(d.inv, nv, N, fb_rows, d_nfb, d.st), kmcudaRuntimeError);
        KNN_CU(launch_knn_search(m, k, d.X, d.C, N, D, K, 0, qlen, d.assign, d.inv, d.off, d.cd, d.radii, d.heap,
                                 d.neigh, d.pairs, fb_rows, d_nfb, d.st), kmcudaRuntimeError);
        KNN_CU(cudaStreamSynchronize(d.st), kmcudaRuntimeError);   // fb_rows goes out of scope
        searched = true;
      } else if (te != cudaSuccess || tc_err) {
        if (shard_tc) {   // the shards cannot be mixed with the exact route: report instead of degrading silently
          KMB_INFO("tensor-core k-NN pass failed on device %d (%s, 0x%x)\n", dev, cudaGetErrorString(te), tc_err);
          return kmcudaRuntimeError;
        }
        KMB_INFO("tensor-core k-NN pass failed (%s, 0x%x): exact search for every query\n", cudaGetErrorString(te), tc_err);
        if (te == cudaErrorMemoryAllocation) cudaGetLastError();
        else if (te != cudaSuccess) { return kmcudaRuntimeError; }
        KNN_CU(cudaMemsetAsync(d.pairs.get(), 0, sizeof(unsigned long long), d.st), kmcudaRuntimeError);
      }
    }
    if (!searched) {
      if (shard_tc) {   // nv < 4096: too few valid samples for the tensor-core pass -- device 0 searches everything exactly
        any_tc_miss = true;
        if (i == 0)
          KNN_CU(launch_knn_search(m, k, d.X, d.C, N, D, K, 0, N, d.assign, d.inv, d.off, d.cd, d.radii, d.heap, d.neigh,
                                   d.pairs, nullptr, nullptr, d.st), kmcudaRuntimeError);
      } else {
        KNN_CU(launch_knn_search(m, k, d.X, d.C, N, D, K, plan[i].first, qlen, d.assign, d.inv, d.off, d.cd,
                                 d.radii, d.heap, d.neigh, d.pairs, nullptr, nullptr, d.st), kmcudaRuntimeError);
      }
    }
    KNN_CU(cudaEventRecord(d.done, d.st), kmcudaRuntimeError);
    return kmcudaSuccess;
  };
#undef KNN_CU
#define KNN_CU(call, code) do { cudaError_t e__ = (call); if (e__ != cudaSuccess) { KMB_INFO("%s:%d -> %s\n", __FILE__, __LINE__, cudaGetErrorString(e__)); cleanup(); return code; } } while (false)
  {
    std::vector<KMCUDAResult> res(dev_ids.size(), kmcudaSuccess);
    if (shard_tc) {
      std::vector<std::thread> workers;
      for (size_t i = 0; i < dev_ids.size(); i++) workers.emplace_back([&, i]() { res[i] = per_device(i); });
      for (auto& w : workers) w.join();
    } else {
      for (size_t i = 0; i < dev_ids.size(); i++) {
        res[i] = per_device(i);
        if (res[i] != kmcudaSuccess) break;
      }
    }
    for (KMCUDAResult r : res)
      if (r != kmcudaSuccess) { cleanup(); return r; }
    if (any_tc_miss) shard_tc_ok = false;
  }
  if (shard_tc) {
    // merge on device 0 (in place): min over the devices' arrays; then one copy-out of all N rows
    KDev& d0 = *kd[0];
    KNN_CU(cudaSetDevice(dev_ids[0]), kmcudaRuntimeError);
    if (shard_tc_ok) {
      PeerU32 pb;
      pb.n = static_cast<int>(dev_ids.size());
      for (size_t i = 0; i < dev_ids.size(); i++) {
        pb.p[i] = kd[i]->neigh.get();
        if (i) KNN_CU(cudaStreamWaitEvent(d0.st, kd[i]->done, 0), kmcudaRuntimeError);
      }
      KNN_CU(launch_peer_min_u32(pb, static_cast<size_t>(N) * k, d0.neigh.get(), d0.st), kmcudaRuntimeError);
    }
    if (device_ptrs < 0)
      KNN_CU(cudaMemcpyAsync(neighbors, d0.neigh.get(), sizeof(uint32_t) * static_cast<size_t>(N) * k,
                             cudaMemcpyDeviceToHost, d0.st), kmcudaMemoryCopyError);
    else
      KNN_CU(cudaMemcpyPeerAsync(neighbors, device_ptrs, d0.neigh.get(), dev_ids[0],
                                 sizeof(uint32_t) * static_cast<size_t>(N) * k, d0.st), kmcudaMemoryCopyError);
  }
  for (size_t i = 0; i < dev_ids.size(); i++) {
    KDev& d = *kd[i];
    const int dev = dev_ids[i];
    const uint32_t qoff = plan[i].first, qlen = plan[i].second;
    KNN_CU(cudaSetDevice(dev), kmcudaRuntimeError);
    if (shard_tc) {
      // (copy-out was issued on device 0 above)
    } else if (device_ptrs < 0)
      KNN_CU(cudaMemcpyAsync(neighbors + static_cast<size_t>(qoff) * k, d.neigh.get(),
                             sizeof(uint32_t) * static_cast<size_t>(qlen) * k, cudaMemcpyDeviceToHost, d.st),
             kmcudaMemoryCopyError);
    else
      KNN_CU(cudaMemcpyPeerAsync(neighbors + static_cast<size_t>(qoff) * k, device_ptrs, d.neigh.get(), dev,
                                 sizeof(uint32_t) * static_cast<size_t>(qlen) * k, d.st), kmcudaMemoryCopyError);
    unsigned long long p = 0;
    KNN_CU(cudaMemcpyAsync(&p, d.pairs.get(), sizeof(p), cudaMemcpyDeviceToHost, d.st), kmcudaMemoryCopyError);
    KNN_CU(cudaStreamSynchronize(d.st), kmcudaRuntimeError);
    total_pairs += p;
  }
#undef KNN_CU
  g_prof.mark("knn: exact search of the remainder + copy-out");
  g_prof.report("knn_cuda");
  cleanup();
  KMB_INFO("calculated %f of all the distances\n",
           static_cast<double>(total_pairs) / (static_cast<double>(N) * N));  // reference knn.cu:530
  KMB_DEBUG("return kmcudaSuccess\n");
  return kmcudaSuccess;
}

}  // extern "C"
