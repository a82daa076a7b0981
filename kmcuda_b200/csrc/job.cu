// job.cu -- the k-means Job (job.h): device setup and the NCCL binding, ingest, the weights check, the centroid update
// and its exchange, the Lloyd / Yinyang / mini-batch loops, the Yinyang grouping and the average distance.
//
// Role of the host halves of the reference's kmeans.cu (Lloyd loop :934-1026, Yinyang loop :1028-1263) and of
// kmcuda.cc's allocation + ingest (:139-170).  Differences by design (DESIGN.md): samples are range-partitioned across
// the GPUs in the mask instead of replicated; no transpose; the per-iteration exchange is ONE NCCL all-reduce of the
// [K][D] partial sums + [K] counts instead of 5-6 rounds of peer copies; centroid update is a deterministic sort +
// segmented compensated sum instead of one thread per centroid.
#include <dlfcn.h>

#include <map>
#include <set>

#include "job.h"

namespace kmb {

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

PhaseProfile g_prof;

KMCUDAResult Job::setup(const std::vector<int>& dev_ids) {
  auto plan = split_rows(N, static_cast<uint32_t>(D) * sizeof(float), dev_ids.size());
  devs = std::vector<Dev>(dev_ids.size());
  for (size_t i = 0; i < dev_ids.size(); i++) {
    Dev& d = devs[i];
    d.dev = dev_ids[i];
    d.off = plan[i].first;
    d.len = plan[i].second;
    KMB_CU(cudaSetDevice(d.dev), kmcudaNoSuchDevice);
    KMB_CU(cudaStreamCreateWithFlags(&d.st, cudaStreamNonBlocking), kmcudaRuntimeError);
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
    if (center_shift) {
      KMB_CU(d.d_shift.alloc(1), kmcudaMemoryAllocationFailure);
      KMB_CU(cudaMemsetAsync(d.d_shift.get(), 0, sizeof(double), d.st), kmcudaRuntimeError);
      if (i == 0) {
        KMB_CU(d.Cold.alloc(static_cast<size_t>(K) * D), kmcudaMemoryAllocationFailure);
        KMB_CU(d.dsq.alloc(K), kmcudaMemoryAllocationFailure);
      }
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
  for (auto& d : devs) {
    KMB_CU(cudaSetDevice(d.dev), kmcudaRuntimeError);
    if (weights) KMB_RET(copy_in(d.w, weights + d.off, d.len, d.dev, device_ptrs, false, d.st, verbosity));
    const float* src = samples + static_cast<size_t>(d.off) * (fp16x2 ? D / 2 : D);
    KMB_RET(copy_in(d.X, src, static_cast<size_t>(d.len) * D, d.dev, device_ptrs, fp16x2, d.st, verbosity));
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
  std::vector<uint32_t> flags;
  std::vector<double> parts;
  KMB_RET(gather([&](size_t i) { return devs[i].d_changed.get(); }, &flags,
                 [&](size_t i) { return devs[i].d_dsum.get(); }, &parts));
  uint32_t bad = 0;
  double total = 0;
  for (size_t i = 0; i < devs.size(); i++) {
    bad |= flags[i];
    total += parts[i];
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

// one assignment pass over every shard; *changed = total reassignments, *shift (if wanted) = the first device's d_shift
KMCUDAResult Job::assign_pass(uint32_t* changed, double* shift) {
  for (auto& d : devs) {
    KMB_CU(cudaSetDevice(d.dev), kmcudaRuntimeError);
    KMB_CU(cudaMemsetAsync(d.d_changed.get(), 0, sizeof(uint32_t), d.st), kmcudaRuntimeError);
    KMB_RET(d.shard->assign(d.len, d.X, d.C, d.assign, d.prev, d.d_changed, d.st));
  }
  std::vector<uint32_t> mine;
  if (shift) {
    std::vector<double> s;
    KMB_RET(gather([&](size_t i) { return devs[i].d_changed.get(); }, &mine,
                   [&](size_t i) { return devs[i].d_shift.get(); }, &s));
    *shift = s[0];
  } else {
    KMB_RET(gather([&](size_t i) { return devs[i].d_changed.get(); }, &mine));
  }
  uint32_t total = 0;
  for (size_t i = 0; i < devs.size(); i++) {
    total += mine[i];
    KMB_RET(devs[i].shard->check_pipeline());
  }
  *changed = total;
  return kmcudaSuccess;
}

// centroid update: shard partial sums -> exchange (peer-memory reduce, or NCCL all-reduce) -> normalise on every GPU
KMCUDAResult Job::update(int iter) {
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
      if (!relocate_empty)
        KMB_RET(d.shard->finish_update(d.rsums, d.rcounts, d.C, d.ccounts, d.st, d.rweights.get(), d.cweights.get()));
    }
    if (!relocate_empty) return kmcudaSuccess;
  }
  if (devs.size() > 1 && !peer_exchange) {
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
  if (relocate_empty) KMB_RET(relocate(iter));
  const bool pe = devs.size() > 1 && peer_exchange;
  for (auto& d : devs) {
    KMB_CU(cudaSetDevice(d.dev), kmcudaRuntimeError);
    if (pe) KMB_RET(d.shard->finish_update(d.rsums, d.rcounts, d.C, d.ccounts, d.st, d.rweights.get(), d.cweights.get()));
    else KMB_RET(d.shard->finish_update(d.sums, d.counts, d.C, d.ccounts, d.st, d.wsums.get(), d.cweights.get()));
    if (metric == 1 && relocated)
      KMB_CU(launch_reloc_cos_overwrite(d.C, D, d.rl_x, d.rl_meta, relocated, d.st), kmcudaRuntimeError);
  }
  return kmcudaSuccess;
}

// Empty-cluster relocation (DESIGN.md §4l), between the exchange and the normalisation: d.C still holds the centroids
// the assignments were made against.  The empty clusters E (exchanged weight total, or count, 0; ascending) take, in
// order, the rows of the walk over (d desc, global row asc) that leave their donor a weight total > 0.  Every device
// offers its top T rows; the merged list is trusted down to the last key of any device that has more eligible rows, and
// T doubles while the walk runs out above that point.  All devices then apply the same records to the same totals.
KMCUDAResult Job::relocate(int iter) {
  relocated = 0;
  const bool pe = devs.size() > 1 && peer_exchange;
  Dev& d0 = devs[0];
  std::vector<float> W(K);
  KMB_CU(cudaSetDevice(d0.dev), kmcudaRuntimeError);
  if (weighted) {
    KMB_CU(cudaMemcpyAsync(W.data(), pe ? d0.rweights.get() : d0.wsums.get(), sizeof(float) * K,
                           cudaMemcpyDeviceToHost, d0.st), kmcudaMemoryCopyError);
    KMB_CU(cudaStreamSynchronize(d0.st), kmcudaRuntimeError);
  } else {
    std::vector<uint32_t> cnt(K);
    KMB_CU(cudaMemcpyAsync(cnt.data(), pe ? d0.rcounts.get() : d0.counts.get(), sizeof(uint32_t) * K,
                           cudaMemcpyDeviceToHost, d0.st), kmcudaMemoryCopyError);
    KMB_CU(cudaStreamSynchronize(d0.st), kmcudaRuntimeError);
    for (uint32_t c = 0; c < K; c++) W[c] = static_cast<float>(cnt[c]);
  }
  std::vector<uint32_t> E;
  for (uint32_t c = 0; c < K; c++)
    if (W[c] == 0) E.push_back(c);
  if (E.empty()) return kmcudaSuccess;
  const uint32_t m = static_cast<uint32_t>(E.size());
  for (auto& d : devs) {
    if (d.len == 0) continue;
    KMB_CU(cudaSetDevice(d.dev), kmcudaRuntimeError);
    if (!d.rl_keys.get()) {
      KMB_CU(d.rl_keys.alloc(d.len), kmcudaMemoryAllocationFailure);
      KMB_CU(d.rl_state.alloc(sizeof(RelocState) / sizeof(uint64_t)), kmcudaMemoryAllocationFailure);
      KMB_CU(d.rl_hist.alloc(256), kmcudaMemoryAllocationFailure);
      KMB_CU(d.rl_nsel.alloc(1), kmcudaMemoryAllocationFailure);
    }
    KMB_CU(launch_reloc_keys(metric, d.X, d.len, D, d.C, K, d.assign, d.w.get(), d.off, d.rl_keys, d.st),
           kmcudaRuntimeError);
  }
  struct Cand {
    uint64_t key;
    uint32_t dev, donor;
    float w;
  };
  std::vector<Cand> taken;
  std::vector<std::vector<uint64_t>> tops(devs.size());
  std::vector<std::vector<uint32_t>> metas(devs.size());
  std::vector<RelocState> states(devs.size());
  for (uint32_t T = 2 * m + 32;; T *= 2) {
    for (size_t i = 0; i < devs.size(); i++) {
      Dev& d = devs[i];
      tops[i].clear();
      if (d.len == 0) continue;
      KMB_CU(cudaSetDevice(d.dev), kmcudaRuntimeError);
      RelocSelect s;
      s.n = d.len;
      s.T = std::min(T, d.len);
      s.cap = reloc_cap(s.T);
      if (s.cap > d.rl_cap) {
        KMB_CU(d.rl_sel.alloc(s.cap), kmcudaMemoryAllocationFailure);
        KMB_CU(d.rl_top.alloc(s.cap), kmcudaMemoryAllocationFailure);
        KMB_CU(d.rl_meta.alloc(2 * static_cast<size_t>(s.cap)), kmcudaMemoryAllocationFailure);
        KMB_CU(d.rl_tmp.alloc(reloc_select_bytes(d.len, s.cap)), kmcudaMemoryAllocationFailure);
        d.rl_cap = s.cap;
      }
      s.keys = d.rl_keys;
      s.state = reinterpret_cast<RelocState*>(d.rl_state.get());
      s.hist = d.rl_hist;
      s.sel = d.rl_sel;
      s.top = d.rl_top;
      s.nsel = d.rl_nsel;
      s.tmp = d.rl_tmp.get();
      s.tmp_bytes = reloc_select_bytes(d.len, s.cap);
      KMB_CU(launch_reloc_select(s, d.st), kmcudaRuntimeError);
      KMB_CU(launch_reloc_gather(d.rl_top, s.T, d.off, d.assign, d.w.get(), d.rl_meta, d.st), kmcudaRuntimeError);
      tops[i].resize(s.T);
      metas[i].resize(2 * static_cast<size_t>(s.T));
      KMB_CU(cudaMemcpyAsync(tops[i].data(), d.rl_top.get(), sizeof(uint64_t) * s.T, cudaMemcpyDeviceToHost, d.st),
             kmcudaMemoryCopyError);
      KMB_CU(cudaMemcpyAsync(metas[i].data(), d.rl_meta.get(), sizeof(uint32_t) * 2 * s.T, cudaMemcpyDeviceToHost,
                             d.st), kmcudaMemoryCopyError);
      KMB_CU(cudaMemcpyAsync(&states[i], s.state, sizeof(RelocState), cudaMemcpyDeviceToHost, d.st),
             kmcudaMemoryCopyError);
    }
    KMB_RET(sync_all());
    std::vector<Cand> list;
    uint64_t cutoff = 0;   // keys below the last one listed by a device with more eligible rows are not trusted
    for (size_t i = 0; i < devs.size(); i++) {
      uint32_t listed = 0;
      for (; listed < tops[i].size() && tops[i][listed]; listed++) {
        float wj;
        memcpy(&wj, &metas[i][2 * listed + 1], sizeof(wj));
        list.push_back({tops[i][listed], static_cast<uint32_t>(i), metas[i][2 * listed], wj});
      }
      if (!tops[i].empty() && states[i].eligible > listed && listed > 0)
        cutoff = std::max(cutoff, tops[i][listed - 1]);
    }
    std::sort(list.begin(), list.end(), [](const Cand& a, const Cand& b) { return a.key > b.key; });
    std::vector<float> Wrun(W);
    taken.clear();
    for (const Cand& c : list) {
      if (c.key < cutoff || taken.size() == m) break;
      const float left = Wrun[c.donor] - c.w;
      if (!(left > 0.f)) continue;   // the donor would be left without weight
      Wrun[c.donor] = left;
      taken.push_back(c);
    }
    if (taken.size() == m || cutoff == 0) break;
  }
  const uint32_t r = static_cast<uint32_t>(taken.size());
  if (r == 0) {
    KMB_INFO("iteration %d: 0 empty clusters relocated, %" PRIu32 " left empty\n", iter, m);
    return kmcudaSuccess;
  }
  // the taken rows, gathered on their devices and broadcast through the host with their records
  std::vector<float> xs(static_cast<size_t>(r) * D);
  std::vector<uint32_t> meta(3 * static_cast<size_t>(r));
  for (uint32_t j = 0; j < r; j++) {
    meta[3 * j] = E[j];
    meta[3 * j + 1] = taken[j].donor;
    memcpy(&meta[3 * j + 2], &taken[j].w, sizeof(float));
  }
  for (auto& d : devs) {
    KMB_CU(cudaSetDevice(d.dev), kmcudaRuntimeError);
    KMB_CU(d.rl_x.alloc(static_cast<size_t>(r) * D), kmcudaMemoryAllocationFailure);
    KMB_CU(d.rl_idx.alloc(r), kmcudaMemoryAllocationFailure);
  }
  for (size_t i = 0; i < devs.size(); i++) {
    Dev& d = devs[i];
    std::vector<uint32_t> pos, idx;
    for (uint32_t j = 0; j < r; j++)
      if (taken[j].dev == i) {
        pos.push_back(j);
        idx.push_back(~static_cast<uint32_t>(taken[j].key) - d.off);
      }
    if (idx.empty()) continue;
    const uint32_t cnt = static_cast<uint32_t>(idx.size());
    std::vector<float> part(static_cast<size_t>(cnt) * D);
    KMB_CU(cudaSetDevice(d.dev), kmcudaRuntimeError);
    KMB_CU(cudaMemcpyAsync(d.rl_idx.get(), idx.data(), sizeof(uint32_t) * cnt, cudaMemcpyHostToDevice, d.st),
           kmcudaMemoryCopyError);
    KMB_CU(launch_kmp_gather(d.X, D, d.rl_idx, cnt, d.rl_x, d.st), kmcudaRuntimeError);
    KMB_CU(cudaMemcpyAsync(part.data(), d.rl_x.get(), sizeof(float) * part.size(), cudaMemcpyDeviceToHost, d.st),
           kmcudaMemoryCopyError);
    KMB_CU(cudaStreamSynchronize(d.st), kmcudaRuntimeError);
    for (uint32_t q = 0; q < cnt; q++)
      std::copy(part.begin() + static_cast<size_t>(q) * D, part.begin() + static_cast<size_t>(q + 1) * D,
                xs.begin() + static_cast<size_t>(pos[q]) * D);
  }
  for (auto& d : devs) {
    KMB_CU(cudaSetDevice(d.dev), kmcudaRuntimeError);
    KMB_CU(d.rl_meta.alloc(std::max<size_t>(3 * static_cast<size_t>(r), 2 * static_cast<size_t>(d.rl_cap))),
           kmcudaMemoryAllocationFailure);
    KMB_CU(cudaMemcpyAsync(d.rl_x.get(), xs.data(), sizeof(float) * xs.size(), cudaMemcpyHostToDevice, d.st),
           kmcudaMemoryCopyError);
    KMB_CU(cudaMemcpyAsync(d.rl_meta.get(), meta.data(), sizeof(uint32_t) * meta.size(), cudaMemcpyHostToDevice,
                           d.st), kmcudaMemoryCopyError);
    if (pe) KMB_CU(launch_reloc_apply(d.rsums, d.rcounts, d.rweights.get(), D, d.rl_x, d.rl_meta, r, d.st),
                   kmcudaRuntimeError);
    else KMB_CU(launch_reloc_apply(d.sums, d.counts, d.wsums.get(), D, d.rl_x, d.rl_meta, r, d.st),
                kmcudaRuntimeError);
  }
  KMB_RET(sync_all());   // the host copies above are pageable and die with this frame
  relocated = r;
  if (r < m) KMB_INFO("iteration %d: %" PRIu32 " empty clusters relocated, %" PRIu32 " left empty\n", iter, r, m - r);
  else KMB_INFO("iteration %d: %" PRIu32 " empty clusters relocated\n", iter, r);
  for (uint32_t j = 0; j < r; j++) {
    const uint32_t ob = static_cast<uint32_t>(taken[j].key >> 32);
    const uint32_t b = (ob & 0x80000000u) ? (ob & 0x7FFFFFFFu) : ~ob;
    float key;
    memcpy(&key, &b, sizeof(key));
    KMB_DEBUG("relocated cluster %" PRIu32 ": sample %" PRIu32 ", key %.9g, donor %" PRIu32 "\n", E[j],
              ~static_cast<uint32_t>(taken[j].key), key, taken[j].donor);
  }
  return kmcudaSuccess;
}

// scikit-learn's _tolerance before its factor tol (DESIGN.md §4p): (sum_f var_f) / D, the unweighted population
// variances of the features, in double.  Each pass sums every shard per feature on its device (launch_col_sums); the
// host adds the devices in device order from 0 and multiplies by 1 / N.  The first pass gives the mean, which goes back
// to every device for the second pass over (x - mean)^2.
KMCUDAResult Job::mean_variance(double* out) {
  const size_t nd = devs.size(), dd = static_cast<size_t>(D);
  std::vector<DevBuf<double>> work(nd), mean(nd), sums(nd);
  Drain drain{*this};
  std::vector<double> part(nd * dd), hmean(dd), var(dd);
  for (int pass = 0; pass < 2; pass++) {
    for (size_t i = 0; i < nd; i++) {
      Dev& d = devs[i];
      KMB_CU(cudaSetDevice(d.dev), kmcudaRuntimeError);
      if (pass == 0) {
        KMB_CU(work[i].alloc(col_sums_doubles(D)), kmcudaMemoryAllocationFailure);
        KMB_CU(mean[i].alloc(dd), kmcudaMemoryAllocationFailure);
        KMB_CU(sums[i].alloc(dd), kmcudaMemoryAllocationFailure);
      } else {
        KMB_CU(cudaMemcpyAsync(mean[i], hmean.data(), sizeof(double) * dd, cudaMemcpyHostToDevice, d.st),
               kmcudaMemoryCopyError);
      }
      KMB_CU(launch_col_sums(d.X, d.len, D, pass ? mean[i].get() : nullptr, work[i], sums[i], d.st),
             kmcudaRuntimeError);
      KMB_CU(cudaMemcpyAsync(part.data() + i * dd, sums[i], sizeof(double) * dd, cudaMemcpyDeviceToHost, d.st),
             kmcudaMemoryCopyError);
    }
    KMB_RET(sync_all());
    std::vector<double>& res = pass ? var : hmean;
    for (size_t f = 0; f < dd; f++) {
      double acc = 0;
      for (size_t i = 0; i < nd; i++) acc += part[i * dd + f];
      res[f] = acc * (1.0 / N);
    }
  }
  double m = 0;
  for (size_t f = 0; f < dd; f++) m += var[f];
  *out = m / D;
  return kmcudaSuccess;
}

// the centre shift of the update that just ran, sum ||C - Cold||^2 on the first device into its d_shift (the host reads
// it back with the next pass); every device holds the same centroids
KMCUDAResult Job::shift_of(const float* Cold) {
  Dev& d = devs[0];
  KMB_CU(cudaSetDevice(d.dev), kmcudaRuntimeError);
  KMB_CU(launch_center_shift(Cold, d.C, K, D, d.dsq, d.d_shift, d.st), kmcudaRuntimeError);
  return kmcudaSuccess;
}

// a Lloyd update; with the rule, the centroids are kept aside first and the shift follows
KMCUDAResult Job::lloyd_update(int iter) {
  Dev& d0 = devs[0];
  if (center_shift) {
    KMB_CU(cudaSetDevice(d0.dev), kmcudaRuntimeError);
    KMB_CU(cudaMemcpyAsync(d0.Cold.get(), d0.C.get(), sizeof(float) * static_cast<size_t>(K) * D,
                           cudaMemcpyDeviceToDevice, d0.st), kmcudaMemoryCopyError);
  }
  KMB_RET(update(iter));
  if (center_shift) KMB_RET(shift_of(d0.Cold));
  g_prof.mark("centroid update");
  return kmcudaSuccess;
}

// scikit-learn's stopping rule (_kmeans_single_lloyd), after pass `iter` with `changed` reassignments; `shift` is the
// centre shift of update iter - 1 (iter > 1), read back with this pass.  The run stops when that update moved the
// centroids by at most shift_tol or was update max_iter (this pass is the final E step, n_iter = iter - 1), else when
// this pass changed no label (n_iter = iter).  Sets n_iter; false without the rule.
bool Job::shift_stop(int iter, uint32_t changed, double shift) {
  if (!center_shift || iter < 2) return false;
  KMB_DEBUG("center shift %d: %.17g (tolerance %.17g)\n", iter - 1, shift, shift_tol);
  const char* why = nullptr;
  int at = iter - 1;
  if (shift <= shift_tol) why = "tolerance";
  else if (at == static_cast<int>(max_iter)) why = "max_iter";
  else if (changed == 0) {
    why = "equal labels";
    at = iter;
  }
  if (!why) return false;
  n_iter = at;
  KMB_INFO("stopped at iteration %d: %s\n", at, why);
  return true;
}

// reference kmeans_cuda_lloyd, kmeans.cu:934-1026.  A fresh run (iter == 0) resets the state and starts with a pass.  A
// run continued after pass `iter` (its assignments belong to the current centroids) starts with the update that is due:
// used when the Yinyang iterations of a run turn out slower than its Lloyd passes (Job::yinyang).
KMCUDAResult Job::lloyd(float tolerance, int iter, int* iter_out, uint32_t* changed_out) {
  if (iter == 0) {
    n_iter = 0;
    for (auto& d : devs) {
      KMB_CU(cudaSetDevice(d.dev), kmcudaRuntimeError);
      KMB_CU(cudaMemsetAsync(d.ccounts.get(), 0, sizeof(uint32_t) * K, d.st), kmcudaRuntimeError);
      if (d.cweights.get()) KMB_CU(cudaMemsetAsync(d.cweights.get(), 0, sizeof(float) * K, d.st), kmcudaRuntimeError);
      KMB_RET(d.shard->reset_update_state(d.st));
      KMB_CU(cudaMemsetAsync(d.assign.get(), 0xff, sizeof(uint32_t) * d.len, d.st), kmcudaRuntimeError);
      KMB_CU(cudaMemsetAsync(d.prev.get(), 0xff, sizeof(uint32_t) * d.len, d.st), kmcudaRuntimeError);
    }
  }
  auto t_prev = std::chrono::steady_clock::now();
  for (;;) {
    if (iter > 0) KMB_RET(lloyd_update(iter));
    iter++;
    uint32_t changed = 0;
    double shift = 0;
    KMB_RET(assign_pass(&changed, center_shift && iter > 1 ? &shift : nullptr));
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
    if (shift_stop(iter, changed, shift)) return kmcudaSuccess;
    if (changed <= tolerance * N) return kmcudaSuccess;  // float compare, kmeans.cu:707
  }
}

// Yinyang groups = k-means (k-means++ with srand(0), Lloyd to 2 %) over the K centroids,
// reference kmeans.cu:1061-1094.  Runs on the first device, result broadcast by the caller.
KMCUDAResult Job::group_centroids(uint32_t G, std::vector<uint32_t>* groups) {
  Job sub(metric, K, D, G, verbosity);
  std::vector<int> one{devs[0].dev};
  KMB_RET(sub.setup(one));
  sub.devs[0].X.borrow(devs[0].C.get());
  srand(0);
  KMB_RET(sub.init_plusplus());
  KMB_INFO("\rdone            \n");
  KMB_RET(sub.lloyd(kYinyangGroupTolerance));
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
    return lloyd(tolerance);
  }
  KMB_INFO("running Lloyd until reassignments drop below %" PRIu32 "\n",
           static_cast<uint32_t>(kYinyangDraftReassignments * N));
  int iter = 0;
  uint32_t changed = 0;
  KMB_RET(lloyd(kYinyangDraftReassignments, 0, &iter, &changed));
  if (n_iter || changed <= tolerance * N) return kmcudaSuccess;   // n_iter: the rule stopped the run in the draft
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
      std::vector<uint32_t> c, p;
      std::vector<double> s(1, 0.0);
      if (center_shift)
        KMB_RET(gather([&](size_t i) { return devs[i].d_changed.get(); }, &c,
                       [&](size_t i) { return devs[i].shard->yy_counters.get() + 1; }, &p,
                       [&](size_t i) { return devs[i].d_shift.get(); }, &s));
      else
        KMB_RET(gather([&](size_t i) { return devs[i].d_changed.get(); }, &c,
                       [&](size_t i) { return devs[i].shard->yy_counters.get() + 1; }, &p));
      uint32_t total_changed = 0, total_passed = 0;
      for (size_t i = 0; i < devs.size(); i++) {
        KMB_RET(devs[i].shard->check_pipeline());
        total_changed += c[i];
        total_passed += p[i];
      }
      KMB_INFO("iteration %d: %" PRIu32 " reassignments\n", iter, total_changed);
      if (shift_stop(iter, total_changed, s[0])) return kmcudaSuccess;
      if (total_changed <= tolerance * N) return kmcudaSuccess;
      {
        const auto t_now = std::chrono::steady_clock::now();
        const double ms = std::chrono::duration<double, std::milli>(t_now - t_prev).count();
        t_prev = t_now;
        if (adaptive && clean && ms > lloyd_iter_ms) {
          KMB_INFO("a Yinyang iteration takes %.2f ms, a Lloyd iteration %.2f ms => Lloyd\n", ms, lloyd_iter_ms);
          return lloyd(tolerance, iter);
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
    KMB_RET(update(iter));
    if (center_shift) KMB_RET(shift_of(devs[0].shard->oldC.get()));
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
  Drain drain{*this};
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
    KMB_RET(mean_variance(&tol_abs));
    tol_abs *= static_cast<double>(tolerance);
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
    KMB_CU(launch_fixed_sum(bsum, nb, stats.get(), d.st), kmcudaRuntimeError);
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

// restart r of restarts() and init r of minibatch_init() seed with seed + r * 0x9E3779B9 (mod 2^32)
static uint32_t restart_seed(uint32_t seed, uint32_t r) { return seed + r * 0x9E3779B9u; }

namespace {
// The best of n runs on the Job's devices (restarts, mini-batch inits) by a value to minimise: run 0 is the first best
// and a later run replaces it only with a strictly lower value, so ties keep the earlier run and NaN never wins.  The
// best run's centroids, and its assignments when they are kept, are copied aside on every device unless it is the last
// run, and restore() copies them back unless the last run is the best.  Declared before the caller's Drain.
struct BestRun {
  Job& job;
  const uint32_t n;
  const int verbosity;   // (KMB_CU's log)
  std::vector<DevBuf<float>> C;
  std::vector<DevBuf<uint32_t>> assign;   // empty when the assignments are not kept
  uint32_t r = 0;
  double value = 0;

  BestRun(Job& job, uint32_t n) : job(job), n(n), verbosity(job.verbosity) {}
  KMCUDAResult alloc(bool with_assign) {
    if (n < 2) return kmcudaSuccess;
    C.resize(job.devs.size());
    if (with_assign) assign.resize(job.devs.size());
    for (size_t i = 0; i < C.size(); i++) {
      KMB_CU(cudaSetDevice(job.devs[i].dev), kmcudaRuntimeError);
      KMB_CU(C[i].alloc(static_cast<size_t>(job.K) * job.D), kmcudaMemoryAllocationFailure);
      if (with_assign) KMB_CU(assign[i].alloc(job.devs[i].len), kmcudaMemoryAllocationFailure);
    }
    return kmcudaSuccess;
  }
  // run `run` ended with `e`; *kept (if wanted): it is the best so far
  KMCUDAResult offer(uint32_t run, double e, bool* kept = nullptr) {
    const bool best = run == 0 || e < value;
    if (kept) *kept = best;
    if (!best) return kmcudaSuccess;
    r = run;
    value = e;
    return run + 1 < n ? copy(true) : kmcudaSuccess;
  }
  KMCUDAResult restore() { return r + 1 < n ? copy(false) : kmcudaSuccess; }

 private:
  template <typename T>
  static cudaError_t copy_one(T* aside_buf, T* live, size_t count, bool aside, cudaStream_t st) {
    return cudaMemcpyAsync(aside ? aside_buf : live, aside ? live : aside_buf, sizeof(T) * count,
                           cudaMemcpyDeviceToDevice, st);
  }
  KMCUDAResult copy(bool aside) {
    for (size_t i = 0; i < C.size(); i++) {
      Dev& d = job.devs[i];
      KMB_CU(cudaSetDevice(d.dev), kmcudaRuntimeError);
      KMB_CU(copy_one(C[i].get(), d.C.get(), static_cast<size_t>(job.K) * job.D, aside, d.st), kmcudaMemoryCopyError);
      if (!assign.empty()) KMB_CU(copy_one(assign[i].get(), d.assign.get(), d.len, aside, d.st), kmcudaMemoryCopyError);
    }
    return kmcudaSuccess;
  }
};
}  // namespace

// The init stage of mini-batch k-means (DESIGN.md §4q), scikit-learn's MiniBatchKMeans init_size / n_init.  Init r seeds
// with seed_r = restart_seed(seed, r), the restart schedule.  When m < N it seeds on the m rows
// floor(u(seed, r, kMbTagInit) * N), drawn with replacement and gathered with their weights into a nested job, which
// runs exactly the seeding of a kmcuda_b200_kmeans_weighted() call on them; otherwise on all rows.  With n_init > 1 the
// inits are ranked by sum w e over m validation rows (kMbTagValid, step 0), assigned by the exact argmin, and the best
// is picked by BestRun.  The kept centroids are left in C.
KMCUDAResult Job::minibatch_init(KMCUDAInitMethod method, const void* init_params, uint32_t seed, uint32_t m,
                                 uint32_t n_init, int device_ptrs, bool fp16x2) {
  Dev& d = devs[0];
  KMB_CU(cudaSetDevice(d.dev), kmcudaRuntimeError);
  const size_t kd = static_cast<size_t>(K) * D;
  const bool subset = m < N;
  DevBuf<uint32_t> rows, vrows, result, row_result, keys;
  DevBuf<float> gx, gw;
  DevBuf<double> bsum, total;
  std::unique_ptr<Shard> vs;   // the validation pass over m row entries
  BestRun best(*this, n_init);
  Drain drain{*this};
  if (subset) {
    KMB_CU(rows.alloc(m), kmcudaMemoryAllocationFailure);
    KMB_CU(gx.alloc(static_cast<size_t>(m) * D), kmcudaMemoryAllocationFailure);
    if (weighted) KMB_CU(gw.alloc(m), kmcudaMemoryAllocationFailure);
  }
  if (n_init > 1) {
    vs.reset(new Shard(metric, d.dev, m, D, K, verbosity));
    KMB_RET(vs->create(false));
    KMB_CU(vrows.alloc(m), kmcudaMemoryAllocationFailure);
    KMB_CU(result.alloc(m), kmcudaMemoryAllocationFailure);
    KMB_CU(row_result.alloc(N), kmcudaMemoryAllocationFailure);
    KMB_CU(keys.alloc(m), kmcudaMemoryAllocationFailure);
    KMB_CU(bsum.alloc(mb_blocks(m)), kmcudaMemoryAllocationFailure);
    KMB_CU(total.alloc(1), kmcudaMemoryAllocationFailure);
    KMB_RET(best.alloc(false));
    KMB_CU(launch_mb_draw(N, m, mb_step_key(seed, 0, kMbTagValid), vrows, d.st), kmcudaRuntimeError);
  }
  for (uint32_t r = 0; r < n_init; r++) {
    const uint32_t seed_r = restart_seed(seed, r);
    // the seeding's own phases stay out of this call's profile
    const bool prof = g_prof.on;
    g_prof.on = false;
    KMCUDAResult res = kmcudaSuccess;
    if (!subset) {
      res = init_centroids(method, init_params, seed_r, device_ptrs, fp16x2, nullptr);
    } else {
      // X (fp16x2 already widened on ingest) and w gathered to [m] rows; the nested job borrows them
      if (cudaSetDevice(d.dev) != cudaSuccess ||
          launch_mb_draw(N, m, mb_step_key(seed, r, kMbTagInit), rows, d.st) != cudaSuccess ||
          launch_kmp_gather(d.X, D, rows, m, gx, d.st) != cudaSuccess ||
          (weighted && launch_kmp_gather(d.w, 1, rows, m, gw, d.st) != cudaSuccess) ||
          cudaStreamSynchronize(d.st) != cudaSuccess)
        res = kmcudaRuntimeError;
      Job sub(metric, m, D, K, verbosity);
      sub.weighted = weighted;
      if (res == kmcudaSuccess) res = sub.setup({d.dev});
      if (res == kmcudaSuccess) {
        sub.devs[0].X.borrow(gx.get());
        if (weighted) {
          sub.devs[0].w.borrow(gw.get());
          res = sub.check_weights();   // (the weights are valid: only their sum over the rows can fail)
          if (res == kmcudaInvalidArguments)
            KMB_INFO("mini-batch init %" PRIu32 "/%" PRIu32 ": the weights of the %" PRIu32 " sampled rows sum to 0\n",
                     r + 1, n_init, m);
        }
      }
      if (res == kmcudaSuccess) res = sub.init_centroids(method, init_params, seed_r, -1, false, nullptr);
      if (res == kmcudaSuccess) res = sub.sync_all();
      if (res == kmcudaSuccess && (cudaSetDevice(d.dev) != cudaSuccess ||
                                   cudaMemcpyAsync(d.C.get(), sub.devs[0].C.get(), sizeof(float) * kd,
                                                   cudaMemcpyDeviceToDevice, d.st) != cudaSuccess ||
                                   cudaStreamSynchronize(d.st) != cudaSuccess))
        res = kmcudaMemoryCopyError;
    }
    g_prof.on = prof;
    KMB_RET(res);
    KMB_CU(cudaSetDevice(d.dev), kmcudaRuntimeError);
    g_prof.mark("mini-batch init: seeding");
    if (n_init == 1) {
      KMB_INFO("mini-batch init %" PRIu32 "/%" PRIu32 ": seed %" PRIu32 ", %" PRIu32 " rows\n", r + 1, n_init, seed_r,
               m);
      break;
    }
    KMB_RET(vs->assign_rows(m, d.X, N, vrows, d.C, row_result, result, d.st));
    KMB_CU(launch_mb_inertia(d.X, vrows, m, D, d.C, K, result, d.w.get(), keys, bsum, d.st), kmcudaRuntimeError);
    KMB_CU(launch_fixed_sum(bsum, mb_blocks(m), total, d.st), kmcudaRuntimeError);
    double e = 0;
    KMB_CU(cudaMemcpyAsync(&e, total.get(), sizeof(double), cudaMemcpyDeviceToHost, d.st), kmcudaMemoryCopyError);
    KMB_CU(cudaStreamSynchronize(d.st), kmcudaRuntimeError);
    KMB_RET(vs->check_pipeline());
    g_prof.mark("mini-batch init: validation");
    KMB_INFO("mini-batch init %" PRIu32 "/%" PRIu32 ": seed %" PRIu32 ", %" PRIu32 " rows, validation inertia %.17g\n",
             r + 1, n_init, seed_r, m, e);
    KMB_RET(best.offer(r, e));
  }
  if (n_init > 1) {
    KMB_RET(best.restore());
    KMB_INFO("mini-batch init: kept init %" PRIu32 "/%" PRIu32 "\n", best.r + 1, n_init);
  }
  return sync_all();
}

// Restarts (DESIGN.md §4n): restart r seeds with restart_seed(seed, r) and runs exactly what a fresh call with that
// seed runs; the samples stay ingested.  State that outlives a run in this Job is reset before each one (the per-device
// update state is reset by lloyd()).  BestRun keeps the run of lowest inertia, its centroids and assignments.
KMCUDAResult Job::restarts(KMCUDAInitMethod method, const void* init_params, uint32_t seed, uint32_t n_init,
                           int device_ptrs, bool fp16x2, const float* user_centroids, float tolerance, uint32_t G,
                           double* inertia_out) {
  BestRun best(*this, n_init);
  Drain drain{*this};
  KMB_RET(best.alloc(true));
  int best_n_iter = 0;
  for (uint32_t r = 0; r < n_init; r++) {
    const uint32_t seed_r = restart_seed(seed, r);
    lloyd_iter_ms = 0;
    relocated = 0;
    KMB_RET(init_centroids(method, init_params, seed_r, device_ptrs, fp16x2, user_centroids));
    g_prof.mark("init centroids");
    KMB_RET(yinyang(tolerance, G));
    if (n_init == 1 && !inertia_out) return kmcudaSuccess;
    double e = 0;
    KMB_RET(inertia(&e));
    g_prof.mark("restarts: inertia");
    if (n_init > 1) KMB_INFO("restart %" PRIu32 "/%" PRIu32 ": seed %" PRIu32 ", inertia %.17g\n", r, n_init, seed_r, e);
    bool kept = false;
    KMB_RET(best.offer(r, e, &kept));
    if (kept) best_n_iter = n_iter;
  }
  KMB_RET(best.restore());
  if (n_init > 1) KMB_INFO("restarts: kept restart %" PRIu32 ", inertia %.17g\n", best.r, best.value);
  n_iter = best_n_iter;
  if (inertia_out) *inertia_out = best.value;
  return kmcudaSuccess;
}

// sum of w e over every shard (launch_inertia), the device totals added in device order
KMCUDAResult Job::inertia(double* out) {
  std::vector<DevBuf<double>> bsum(devs.size()), total(devs.size());
  Drain drain{*this};
  for (size_t i = 0; i < devs.size(); i++) {
    Dev& d = devs[i];
    KMB_CU(cudaSetDevice(d.dev), kmcudaRuntimeError);
    KMB_CU(bsum[i].alloc(inertia_blocks(d.len)), kmcudaMemoryAllocationFailure);
    KMB_CU(total[i].alloc(1), kmcudaMemoryAllocationFailure);
    KMB_CU(launch_inertia(metric, d.X, d.len, D, d.C, K, d.assign, d.w.get(), bsum[i], total[i], d.st),
           kmcudaRuntimeError);
  }
  std::vector<double> parts;
  KMB_RET(gather([&](size_t i) { return total[i].get(); }, &parts));
  double sum = 0;
  for (double part : parts) sum += part;
  *out = sum;
  return kmcudaSuccess;
}

KMCUDAResult Job::average_distance(float* out) {
  KMB_INFO("calculating the average distance...\n");
  for (auto& d : devs) {
    KMB_CU(cudaSetDevice(d.dev), kmcudaRuntimeError);
    KMB_CU(cudaMemsetAsync(d.d_dsum.get(), 0, sizeof(double), d.st), kmcudaRuntimeError);
    KMB_CU(launch_average_distance(metric, d.X, d.C, d.len, D, d.assign, d.d_dsum, d.st, d.w.get()), kmcudaRuntimeError);
  }
  std::vector<double> parts;
  KMB_RET(gather([&](size_t i) { return devs[i].d_dsum.get(); }, &parts));
  double sum = 0;
  for (double part : parts) sum += part;
  *out = static_cast<float>(sum / (weighted ? wtotal : N));   // weighted: sum w d / sum w
  return kmcudaSuccess;
}
// Bisecting k-means (DESIGN.md §4o): scikit-learn's BisectingKMeans with this library's draws and fixed-order sums, on
// one GPU.  The leaves are ranges of perm; each round splits the pickable leaf of largest score (lowest lo on ties).  A
// node's bisection depends on its rows and range only, so the host bisects ahead: when the top pickable leaf has no
// cached result, one wave bisects every uncached leaf among the top K - #leaves, all n_init inits of all of them in the
// same launches, and the rounds then apply cached results in pick order.  Nodes bisected but never picked are the waste;
// a wave holds at most K - #leaves nodes.  Every wave-iteration reads the status records back in one copy.
KMCUDAResult Job::bisecting(uint32_t seed, float tolerance, int strategy, uint32_t n_init, uint32_t trials,
                            double* inertia_out) {
  static const char* const kStop[] = {"equal labels", "tolerance", "max_iter"};
  Dev& d = devs[0];
  KMB_CU(cudaSetDevice(d.dev), kmcudaRuntimeError);
  Drain drain{*this};
  // scikit-learn's KMeans _tolerance (BisectingKMeans 1.9 passes tol unscaled): tolerance times the mean of the
  // unweighted per-feature variances; a non-finite sample makes that mean non-finite
  double tol_abs = 0;
  KMB_RET(mean_variance(&tol_abs));
  if (!std::isfinite(tol_abs)) {
    KMB_INFO("bisecting k-means takes finite samples\n");
    return kmcudaInvalidArguments;
  }
  tol_abs *= static_cast<double>(tolerance);
  // a wave's segments of one init are disjoint ranges; segment, slot and chunk indices are 32-bit and the chunks are one
  // grid, so a call whose n_init * K does not fit is rejected
  const size_t nch_max = static_cast<size_t>(n_init) * (cdiv(N, kBkChunk) + static_cast<size_t>(K));
  const size_t nseg_max = static_cast<size_t>(n_init) * K;
  if (2 * nseg_max > UINT32_MAX || nch_max > INT32_MAX) {
    KMB_INFO("bisecting k-means: n_init * clusters is too large\n");
    return kmcudaInvalidArguments;
  }
  DevBuf<uint32_t> perm, perm2, flags, excl, leaf_lo;
  DevBuf<uint8_t> lab;
  DevBuf<BkSeg> segs;
  DevBuf<uint2> work;
  DevBuf<float> cbuf, csq;
  DevBuf<double> part;
  DevBuf<BkChunkStat> cstat;
  DevBuf<BkKey> keys;
  DevBuf<BkStatus> status;
  DevBuf<char> tmp;
  DevBuf<float> dist;
  DevBuf<BkKey> tkeys;
  DevBuf<double> phi;
  DevBuf<uint32_t> trows;
  if (trials) {   // greedy init
    KMB_CU(dist.alloc(static_cast<size_t>(n_init) * N), kmcudaMemoryAllocationFailure);
    KMB_CU(tkeys.alloc(nch_max * kGppMaxTrials), kmcudaMemoryAllocationFailure);
    KMB_CU(phi.alloc(nch_max * kGppMaxTrials), kmcudaMemoryAllocationFailure);
    KMB_CU(trows.alloc(nseg_max * kGppMaxTrials), kmcudaMemoryAllocationFailure);
  }
  const size_t tmp_bytes = bk_split_bytes(N);
  KMB_CU(perm.alloc(N), kmcudaMemoryAllocationFailure);
  KMB_CU(perm2.alloc(N), kmcudaMemoryAllocationFailure);
  KMB_CU(flags.alloc(N + 1), kmcudaMemoryAllocationFailure);
  KMB_CU(excl.alloc(N + 1), kmcudaMemoryAllocationFailure);
  KMB_CU(leaf_lo.alloc(K), kmcudaMemoryAllocationFailure);
  KMB_CU(lab.alloc(static_cast<size_t>(n_init) * N), kmcudaMemoryAllocationFailure);
  KMB_CU(segs.alloc(nseg_max), kmcudaMemoryAllocationFailure);
  KMB_CU(work.alloc(nch_max), kmcudaMemoryAllocationFailure);
  KMB_CU(cbuf.alloc(static_cast<size_t>(nseg_max) * 4 * D), kmcudaMemoryAllocationFailure);
  KMB_CU(csq.alloc(static_cast<size_t>(nseg_max) * 4), kmcudaMemoryAllocationFailure);
  KMB_CU(part.alloc(static_cast<size_t>(nch_max) * bk_partial_doubles(D)), kmcudaMemoryAllocationFailure);
  KMB_CU(cstat.alloc(nch_max), kmcudaMemoryAllocationFailure);
  KMB_CU(keys.alloc(2 * static_cast<size_t>(nch_max)), kmcudaMemoryAllocationFailure);
  KMB_CU(status.alloc(nseg_max), kmcudaMemoryAllocationFailure);
  KMB_CU(tmp.alloc(tmp_bytes), kmcudaMemoryAllocationFailure);
  KMB_CU(launch_bk_iota(perm, N, d.st), kmcudaRuntimeError);
  BkLaunch la;
  la.X = d.X;
  la.D = D;
  la.N = N;
  la.w = d.w.get();
  la.lab = lab;
  la.segs = segs;
  la.work = work;
  la.cbuf = cbuf;
  la.csq = csq;
  la.part = part;
  la.cstat = cstat;
  la.keys = keys;
  la.dist = dist.get();
  la.tkeys = tkeys.get();
  la.phi = phi.get();
  la.trows = trows.get();
  la.status = status;
  uint32_t* cur_perm = perm.get();
  uint32_t* alt_perm = perm2.get();
  g_prof.mark("bisecting: setup");

  struct Result {
    bool splittable;
    uint32_t r, n0;
    double score[2];
    std::vector<float> C;   // [2][D]
  };
  std::map<uint32_t, uint32_t> leaves;              // lo -> hi of every leaf, in perm order
  std::map<uint32_t, std::vector<float>> centre;    // lo -> centre of the leaf
  auto order = [](const std::pair<double, uint32_t>& a, const std::pair<double, uint32_t>& b) {
    return a.first > b.first || (a.first == b.first && a.second < b.second);
  };
  std::set<std::pair<double, uint32_t>, decltype(order)> pickable(order);   // (score, lo)
  std::map<uint32_t, Result> cache;                  // lo of a leaf -> its bisection
  std::vector<BkSeg> pending;                        // splits decided but not yet applied to perm
  leaves[0] = N;
  pickable.insert({0.0, 0u});
  uint32_t waves = 0, bisected = 0;
  std::vector<BkSeg> hs;
  std::vector<uint2> hw;
  std::vector<BkStatus> hst;
  // the table of CTAs for the segments hs: {segment, chunk} pairs
  auto upload = [&](bool with_work) -> KMCUDAResult {
    if (with_work) {
      hw.clear();
      for (uint32_t s = 0; s < hs.size(); s++)
        for (uint32_t c = 0; c < cdiv(hs[s].hi - hs[s].lo, kBkChunk); c++) hw.push_back({s, c});
      KMB_CU(cudaMemcpyAsync(work.get(), hw.data(), sizeof(uint2) * hw.size(), cudaMemcpyHostToDevice, d.st),
             kmcudaMemoryCopyError);
    }
    KMB_CU(cudaMemcpyAsync(segs.get(), hs.data(), sizeof(BkSeg) * hs.size(), cudaMemcpyHostToDevice, d.st),
           kmcudaMemoryCopyError);
    la.nseg = static_cast<uint32_t>(hs.size());
    la.nwork = static_cast<uint32_t>(hw.size());
    la.perm = cur_perm;
    return kmcudaSuccess;
  };
  auto read_status = [&]() -> KMCUDAResult {
    hst.resize(hs.size());
    KMB_CU(cudaMemcpyAsync(hst.data(), status.get(), sizeof(BkStatus) * hs.size(), cudaMemcpyDeviceToHost, d.st),
           kmcudaMemoryCopyError);
    KMB_CU(cudaStreamSynchronize(d.st), kmcudaRuntimeError);
    return kmcudaSuccess;
  };
  auto apply_pending = [&]() -> KMCUDAResult {
    if (pending.empty()) return kmcudaSuccess;
    hs = pending;
    pending.clear();
    KMB_RET(upload(true));
    KMB_CU(launch_bk_split(la, flags, excl, tmp.get(), tmp_bytes, alt_perm, d.st), kmcudaRuntimeError);
    std::swap(cur_perm, alt_perm);
    g_prof.mark("bisecting: split");
    return kmcudaSuccess;
  };
  // bisects the nodes [lo, hi) of `nodes` (one segment per node and init) into the cache
  auto wave = [&](const std::vector<std::pair<uint32_t, uint32_t>>& nodes) -> KMCUDAResult {
    waves++;
    bisected += static_cast<uint32_t>(nodes.size());
    hs.clear();
    uint32_t pbase = 0;
    for (auto& nd : nodes)
      for (uint32_t r = 0; r < n_init; r++) {
        const uint32_t s = static_cast<uint32_t>(hs.size());
        hs.push_back({nd.first, nd.second, r, kBkRun, 2 * s, 2 * s + 1, pbase, seed,
                      bk_node_key(seed, nd.first, nd.second, r, 0)});
        pbase += cdiv(nd.second - nd.first, kBkChunk);
      }
    const std::vector<BkSeg> all = hs;
    KMB_RET(upload(true));
    KMB_CU(launch_bk_init(la, trials, d.st), kmcudaRuntimeError);
    KMB_RET(read_status());
    g_prof.mark("bisecting: init");
    const size_t ns = all.size();
    std::vector<BkStatus> fin(ns);
    std::vector<uint32_t> iters(ns, 0), cur_slot(ns), stop(ns, 0);
    std::vector<char> done(ns, 0), noinit(ns, 0);
    std::vector<uint32_t> active;
    for (uint32_t s = 0; s < ns; s++) {
      cur_slot[s] = all[s].cur;
      if (hst[s].init_row[1] == UINT32_MAX) {
        noinit[s] = 1;
        done[s] = 1;
      } else {
        active.push_back(s);
      }
    }
    std::vector<uint32_t> mode(ns, kBkRun);
    while (!active.empty()) {
      hs.clear();
      for (uint32_t s : active) {
        BkSeg g = all[s];
        g.mode = mode[s];
        g.cur = cur_slot[s];
        g.nxt = cur_slot[s] ^ 1u;
        hs.push_back(g);
      }
      KMB_RET(upload(true));
      KMB_CU(launch_bk_step(la, d.st), kmcudaRuntimeError);
      KMB_RET(read_status());
      std::vector<uint32_t> next;
      for (size_t a = 0; a < active.size(); a++) {
        const uint32_t s = active[a];
        const BkStatus& st = hst[a];
        if (mode[s] == kBkFinal) {
          fin[s] = st;
          done[s] = 1;
          continue;
        }
        const uint32_t i = iters[s]++;
        if (i > 0 && st.changed == 0) {   // strict convergence: the labels and centres of this E step stand
          fin[s] = st;
          done[s] = 1;
          stop[s] = 0;
          continue;
        }
        cur_slot[s] ^= 1u;
        if (st.shift <= tol_abs) {
          mode[s] = kBkFinal;
          stop[s] = 1;
        } else if (iters[s] == max_iter) {
          mode[s] = kBkFinal;
          stop[s] = 2;
        }
        next.push_back(s);
      }
      active.swap(next);
    }
    g_prof.mark("bisecting: 2-means");
    std::vector<float> hc(static_cast<size_t>(ns) * 4 * D);
    KMB_CU(cudaMemcpyAsync(hc.data(), cbuf.get(), sizeof(float) * hc.size(), cudaMemcpyDeviceToHost, d.st),
           kmcudaMemoryCopyError);
    KMB_CU(cudaStreamSynchronize(d.st), kmcudaRuntimeError);
    for (size_t b = 0; b < ns; b += n_init) {
      const uint32_t lo = all[b].lo, hi = all[b].hi;
      Result res{false, 0, 0, {0, 0}, {}};
      if (noinit[b]) {
        KMB_DEBUG("bisecting: node [%" PRIu32 ", %" PRIu32 ") has no init\n", lo, hi);
      } else {
        uint32_t best = 0;
        for (uint32_t r = 0; r < n_init; r++) {
          const BkStatus& st = fin[b + r];
          KMB_DEBUG("bisecting: node [%" PRIu32 ", %" PRIu32 ") init %" PRIu32 ": %" PRIu32
                    " iterations, stopped on %s, inertia %.17g\n", lo, hi, r, iters[b + r], kStop[stop[b + r]],
                    st.inertia);
          if (r > 0 && st.inertia < fin[b + best].inertia * (1 - 1e-6)) best = r;   // scikit-learn's _bisect
        }
        const BkStatus& st = fin[b + best];
        res.splittable = st.W[0] > 0 && st.W[1] > 0;
        res.r = best;
        res.n0 = st.cnt[0];
        for (int j = 0; j < 2; j++) res.score[j] = strategy == 0 ? st.I[j] : static_cast<double>(st.cnt[j]);
        const float* c = hc.data() + static_cast<size_t>(cur_slot[b + best]) * 2 * D;
        res.C.assign(c, c + 2 * D);
      }
      cache[lo] = std::move(res);
    }
    return kmcudaSuccess;
  };

  uint32_t nleaves = 1;
  while (nleaves < K) {
    if (pickable.empty()) {
      KMB_INFO("bisecting: only %" PRIu32 " of %" PRIu32 " clusters can be made from these samples\n", nleaves, K);
      return kmcudaInvalidArguments;
    }
    const auto top = *pickable.begin();
    const uint32_t lo = top.second, hi = leaves[lo];
    auto it = cache.find(lo);
    if (it == cache.end()) {
      KMB_RET(apply_pending());
      std::vector<std::pair<uint32_t, uint32_t>> nodes;
      uint32_t taken = 0;
      for (auto p = pickable.begin(); p != pickable.end() && taken < K - nleaves; ++p, ++taken)
        if (!cache.count(p->second)) nodes.push_back({p->second, leaves[p->second]});
      KMB_RET(wave(nodes));
      continue;
    }
    Result res = std::move(it->second);
    cache.erase(it);
    pickable.erase(pickable.begin());
    if (!res.splittable) {
      KMB_INFO("bisecting: [%" PRIu32 ", %" PRIu32 ") is not split\n", lo, hi);
      continue;
    }
    const uint32_t mid = lo + res.n0;
    KMB_INFO("bisecting: split [%" PRIu32 ", %" PRIu32 ") into %" PRIu32 " + %" PRIu32 " rows, scores %.17g %.17g\n", lo,
             hi, res.n0, hi - mid, res.score[0], res.score[1]);
    pending.push_back({lo, hi, res.r, 0, 0, 0, 0, 0, 0});
    leaves[lo] = mid;
    leaves[mid] = hi;
    centre[lo].assign(res.C.begin(), res.C.begin() + D);
    centre[mid].assign(res.C.begin() + D, res.C.end());
    pickable.insert({res.score[0], lo});
    pickable.insert({res.score[1], mid});
    nleaves++;
  }
  KMB_RET(apply_pending());
  std::vector<uint32_t> hlo;
  std::vector<float> hC;
  hlo.reserve(K);
  hC.reserve(static_cast<size_t>(K) * D);
  for (auto& lf : leaves) {
    hlo.push_back(lf.first);
    hC.insert(hC.end(), centre[lf.first].begin(), centre[lf.first].end());
  }
  KMB_CU(cudaMemcpyAsync(leaf_lo.get(), hlo.data(), sizeof(uint32_t) * K, cudaMemcpyHostToDevice, d.st),
         kmcudaMemoryCopyError);
  KMB_CU(cudaMemcpyAsync(d.C.get(), hC.data(), sizeof(float) * hC.size(), cudaMemcpyHostToDevice, d.st),
         kmcudaMemoryCopyError);
  KMB_CU(launch_bk_assign(cur_perm, N, leaf_lo, K, d.assign, d.st), kmcudaRuntimeError);
  KMB_CU(cudaStreamSynchronize(d.st), kmcudaRuntimeError);
  g_prof.mark("bisecting: labels");
  double e = 0;
  if (inertia_out || verbosity > 0) KMB_RET(inertia(&e));
  KMB_INFO("bisecting: %" PRIu32 " waves, %" PRIu32 " nodes bisected, inertia %.17g\n", waves, bisected, e);
  if (inertia_out) *inertia_out = e;
  return kmcudaSuccess;
}
}  // namespace kmb
