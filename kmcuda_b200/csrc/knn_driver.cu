// knn_driver.cu -- knn_cuda() after its argument checks (reference kmcuda.cc:572-730): per-device ingest and search, the
// merge of sharded results, the copy-out.
#include <atomic>
#include <thread>

#include "job.h"

namespace kmb {
namespace {

// one device's k-NN state; owns its stream and event (never copied or moved)
struct KDev {
  int dev = 0;
  DevBuf<float> X, C, cd, radii, heap;
  DevBuf<float> cd_l2, radii_l2;   // angular metric on the tensor-core route: its cluster pruning works in L2
  DevBuf<uint32_t> assign, inv_keys, iota, inv, off, counts, neigh;
  DevBuf<char> cub;
  DevBuf<unsigned long long> pairs;
  cudaStream_t st = nullptr;
  cudaEvent_t done = nullptr;

  explicit KDev(int dev) : dev(dev) {}
  KDev(const KDev&) = delete;
  KDev& operator=(const KDev&) = delete;
  ~KDev() { retire_stream(dev, st, {done}); }
};

// Device i's pipeline: ingest, inverse assignments, radii, centroid distances, then the search of its queries `rows`
// (offset, length: the exact route); ends with d.done recorded on d.st.  Every device gets the whole sample matrix
// (candidates can live anywhere) and its slice of queries.  tc: the tensor-core candidate search applies; shard_tc:
// several GPUs share it.
KMCUDAResult knn_device(size_t i, KDev& d, uint16_t k, int m, uint32_t N, int D, uint32_t K, size_t ndev,
                        int32_t device_ptrs, bool fp16x2, int verbosity, const float* samples, const float* centroids,
                        const uint32_t* assignments, std::pair<uint32_t, uint32_t> rows, bool tc, bool shard_tc,
                        std::atomic<bool>* any_tc_miss) {
  const int dev = d.dev;
  const uint32_t qlen = shard_tc ? N : rows.second;   // rows of this device's neighbour array
  KMB_CU(cudaSetDevice(dev), kmcudaNoSuchDevice);
  KMB_CU(cudaStreamCreateWithFlags(&d.st, cudaStreamNonBlocking), kmcudaRuntimeError);
  KMB_CU(cudaEventCreateWithFlags(&d.done, cudaEventDisableTiming), kmcudaRuntimeError);
  const size_t xcount = static_cast<size_t>(N) * D, ccount = static_cast<size_t>(K) * D;
  if (copy_in(d.X, samples, xcount, dev, device_ptrs, fp16x2, d.st, verbosity) != kmcudaSuccess ||
      copy_in(d.C, centroids, ccount, dev, device_ptrs, fp16x2, d.st, verbosity) != kmcudaSuccess)
    return kmcudaMemoryCopyError;
  KMB_RET(copy_in(d.assign, assignments, N, dev, device_ptrs, false, d.st, verbosity, true, false));
  KMB_CU(d.inv_keys.alloc(N), kmcudaMemoryAllocationFailure);
  KMB_CU(d.iota.alloc(N), kmcudaMemoryAllocationFailure);
  KMB_CU(d.inv.alloc(N), kmcudaMemoryAllocationFailure);
  KMB_CU(d.off.alloc(static_cast<size_t>(K) + 1), kmcudaMemoryAllocationFailure);
  KMB_CU(d.counts.alloc(K), kmcudaMemoryAllocationFailure);
  KMB_CU(d.cd.alloc(static_cast<size_t>(K) * K), kmcudaMemoryAllocationFailure);
  KMB_CU(d.radii.alloc(K), kmcudaMemoryAllocationFailure);
  KMB_CU(d.heap.alloc(static_cast<size_t>(qlen) * 2 * k), kmcudaMemoryAllocationFailure);
  KMB_CU(d.neigh.alloc(static_cast<size_t>(qlen) * k), kmcudaMemoryAllocationFailure);
  KMB_CU(d.pairs.alloc(1), kmcudaMemoryAllocationFailure);
  KMB_CU(cudaMemsetAsync(d.pairs.get(), 0, sizeof(unsigned long long), d.st), kmcudaRuntimeError);
  if (shard_tc) KMB_CU(cudaMemsetAsync(d.neigh.get(), 0xff, sizeof(uint32_t) * static_cast<size_t>(qlen) * k, d.st), kmcudaRuntimeError);
  // inverse assignments (reference: host std::sort of (assignment, index) tuples, kmcuda.cc:648-691):
  // stable device radix sort + binary-searched CSR offsets
  if (i == 0) KMB_INFO("initializing the inverse assignments...\n");
  UpdateWorkspace ws;
  ws.cub_tmp_bytes = update_cub_bytes(N);
  KMB_CU(d.cub.alloc(ws.cub_tmp_bytes), kmcudaMemoryAllocationFailure);
  ws.cub_tmp = d.cub.get();
  if (ndev == 1) g_prof.mark("knn: alloc + ingest");
  KMB_CU(launch_knn_inverse(d.assign, N, K, d.iota, d.inv_keys, d.inv, d.off, d.counts, ws, d.st), kmcudaRuntimeError);
  KMB_CU(launch_knn_radii(m, d.X, d.C, N, D, K, d.assign, d.radii, d.st), kmcudaRuntimeError);
  KMB_CU(launch_knn_centroid_distances(m, d.C, K, D, d.cd, d.st), kmcudaRuntimeError);
  KMB_CU(launch_knn_radii_fix(d.off, K, d.radii, d.st), kmcudaRuntimeError);
  if (ndev == 1) g_prof.mark("knn: inverse, radii, centroid distances");
  bool searched = false;
  if (tc && (ndev == 1 || shard_tc)) {
    // tensor-core candidate search; the rows it cannot serve go through the reference-order search below
    uint32_t nv = 0, tc_err = 0;
    KMB_CU(cudaMemcpyAsync(&nv, d.off.get() + K, sizeof(nv), cudaMemcpyDeviceToHost, d.st), kmcudaMemoryCopyError);
    KMB_CU(cudaStreamSynchronize(d.st), kmcudaRuntimeError);
    DevBuf<uint32_t> fb_rows, d_nfb;
    KMB_CU(fb_rows.alloc(N), kmcudaMemoryAllocationFailure);
    KMB_CU(d_nfb.alloc(1), kmcudaMemoryAllocationFailure);
    KMB_CU(cudaMemsetAsync(d_nfb.get(), 0, sizeof(uint32_t), d.st), kmcudaRuntimeError);
    cudaError_t te = cudaSuccess;
    const float *tcd = d.cd, *tradii = d.radii;
    if (m == 1 && nv >= 4096) {
      KMB_CU(d.cd_l2.alloc(static_cast<size_t>(K) * K), kmcudaMemoryAllocationFailure);
      KMB_CU(d.radii_l2.alloc(K), kmcudaMemoryAllocationFailure);
      KMB_CU(launch_knn_radii(0, d.X, d.C, N, D, K, d.assign, d.radii_l2, d.st), kmcudaRuntimeError);
      KMB_CU(launch_knn_centroid_distances(0, d.C, K, D, d.cd_l2, d.st), kmcudaRuntimeError);
      KMB_CU(launch_knn_radii_fix(d.off, K, d.radii_l2, d.st), kmcudaRuntimeError);
      tcd = d.cd_l2;
      tradii = d.radii_l2;
    }
    if (nv >= 4096)
      te = tc_knn_search(m, k, d.X, d.C, N, D, K, d.assign, d.inv, d.off, tcd, tradii, nv, d.neigh, fb_rows, d_nfb,
                         d.pairs, &tc_err, shard_tc ? static_cast<uint32_t>(i) : 0u,
                         shard_tc ? static_cast<uint32_t>(ndev) : 1u, d.st);
    if (ndev == 1) g_prof.mark("knn: tensor-core candidate search");
    if (nv >= 4096 && te == cudaSuccess && tc_err == 0) {
      if (i == 0) KMB_CU(launch_knn_tail_rows(d.inv, nv, N, fb_rows, d_nfb, d.st), kmcudaRuntimeError);
      KMB_CU(launch_knn_search(m, k, d.X, d.C, N, D, K, 0, qlen, d.assign, d.inv, d.off, d.cd, d.radii, d.heap,
                               d.neigh, d.pairs, fb_rows, d_nfb, d.st), kmcudaRuntimeError);
      KMB_CU(cudaStreamSynchronize(d.st), kmcudaRuntimeError);   // fb_rows goes out of scope
      searched = true;
    } else if (te != cudaSuccess || tc_err) {
      if (shard_tc) {   // the shards cannot be mixed with the exact route: report instead of degrading silently
        KMB_INFO("tensor-core k-NN pass failed on device %d (%s, 0x%x)\n", dev, cudaGetErrorString(te), tc_err);
        return kmcudaRuntimeError;
      }
      KMB_INFO("tensor-core k-NN pass failed (%s, 0x%x): exact search for every query\n", cudaGetErrorString(te), tc_err);
      if (te == cudaErrorMemoryAllocation) cudaGetLastError();
      else if (te != cudaSuccess) { return kmcudaRuntimeError; }
      KMB_CU(cudaMemsetAsync(d.pairs.get(), 0, sizeof(unsigned long long), d.st), kmcudaRuntimeError);
    }
  }
  if (!searched) {
    if (shard_tc) {   // nv < 4096: too few valid samples for the tensor-core pass -- device 0 searches everything exactly
      *any_tc_miss = true;
      if (i == 0)
        KMB_CU(launch_knn_search(m, k, d.X, d.C, N, D, K, 0, N, d.assign, d.inv, d.off, d.cd, d.radii, d.heap, d.neigh,
                                 d.pairs, nullptr, nullptr, d.st), kmcudaRuntimeError);
    } else {
      KMB_CU(launch_knn_search(m, k, d.X, d.C, N, D, K, rows.first, qlen, d.assign, d.inv, d.off, d.cd,
                               d.radii, d.heap, d.neigh, d.pairs, nullptr, nullptr, d.st), kmcudaRuntimeError);
    }
  }
  KMB_CU(cudaEventRecord(d.done, d.st), kmcudaRuntimeError);
  return kmcudaSuccess;
}

}  // namespace

KMCUDAResult knn_run(uint16_t k, int metric, uint32_t N, int D, uint32_t K, const std::vector<int>& dev_ids,
                     int32_t device_ptrs, bool fp16x2, int verbosity, const float* samples, const float* centroids,
                     const uint32_t* assignments, uint32_t* neighbors) {
  const char* fx = getenv("KMCUDA_B200_FORCE_EXACT");
  const bool tc = !(fx && fx[0] == '1') && tc_knn_supported(metric, k, N, D, K);
  // Several GPUs on the tensor-core path: every GPU holds all samples (as in the reference, kmcuda.cc:157-158) and
  // the cluster-aligned candidate table, and serves an equal share of the query TILES into its own full-size
  // neighbour array; device 0 merges the arrays over peer memory (element-wise minimum against the 0xFFFFFFFF fill).
  bool shard_tc = dev_ids.size() > 1 && metric == 0 && tc;
  for (size_t i = 0; i < dev_ids.size() && shard_tc; i++)
    for (size_t j = 0; j < dev_ids.size() && shard_tc; j++) {
      int access = 0;
      if (i != j && (cudaDeviceCanAccessPeer(&access, dev_ids[i], dev_ids[j]) != cudaSuccess || !access)) shard_tc = false;
    }
  const auto plan = split_rows(N, static_cast<uint32_t>(D) * sizeof(float), dev_ids.size());
  std::atomic<bool> any_tc_miss{false};
  g_prof.begin(dev_ids);
  std::vector<std::unique_ptr<KDev>> kd;
  for (int dev : dev_ids) kd.emplace_back(new KDev(dev));
  // device 0's stream reads every device's neighbour array (the merge): all streams drain before any buffer is released
  struct DrainAll {
    std::vector<std::unique_ptr<KDev>>& kd;
    ~DrainAll() { for (auto& d : kd) sync_stream(d->dev, d->st); }
  } drain_all{kd};
  auto search = [&](size_t i) {
    return knn_device(i, *kd[i], k, metric, N, D, K, dev_ids.size(), device_ptrs, fp16x2, verbosity, samples, centroids,
                      assignments, plan[i], tc, shard_tc, &any_tc_miss);
  };
  {
    // with several devices on the tensor-core path the per-device pipelines (which synchronise their own stream a few
    // times) run on one host thread each, so the GPUs work concurrently
    std::vector<KMCUDAResult> res(dev_ids.size(), kmcudaSuccess);
    if (shard_tc) {
      std::vector<std::thread> workers;
      for (size_t i = 0; i < dev_ids.size(); i++) workers.emplace_back([&, i]() { res[i] = search(i); });
      for (auto& w : workers) w.join();
    } else {
      for (size_t i = 0; i < dev_ids.size(); i++) {
        res[i] = search(i);
        if (res[i] != kmcudaSuccess) break;
      }
    }
    for (KMCUDAResult r : res) KMB_RET(r);
  }
  const size_t nk = static_cast<size_t>(N) * k;
  if (shard_tc) {
    // merge on device 0 (in place): min over the devices' arrays; then one copy-out of all N rows
    KDev& d0 = *kd[0];
    KMB_CU(cudaSetDevice(d0.dev), kmcudaRuntimeError);
    if (!any_tc_miss) {
      PeerU32 pb;
      pb.n = static_cast<int>(dev_ids.size());
      for (size_t i = 0; i < dev_ids.size(); i++) {
        pb.p[i] = kd[i]->neigh.get();
        if (i) KMB_CU(cudaStreamWaitEvent(d0.st, kd[i]->done, 0), kmcudaRuntimeError);
      }
      KMB_CU(launch_peer_min_u32(pb, nk, d0.neigh.get(), d0.st), kmcudaRuntimeError);
    }
    KMB_RET(copy_out(neighbors, d0.neigh.get(), nk, d0.dev, device_ptrs, false, d0.st, verbosity));
  }
  unsigned long long total_pairs = 0;
  for (size_t i = 0; i < dev_ids.size(); i++) {
    KDev& d = *kd[i];
    KMB_CU(cudaSetDevice(d.dev), kmcudaRuntimeError);
    if (!shard_tc)   // (with shard_tc the copy-out was issued on device 0 above)
      KMB_RET(copy_out(neighbors + static_cast<size_t>(plan[i].first) * k, d.neigh.get(),
                       static_cast<size_t>(plan[i].second) * k, d.dev, device_ptrs, false, d.st, verbosity));
    unsigned long long p = 0;
    KMB_CU(cudaMemcpyAsync(&p, d.pairs.get(), sizeof(p), cudaMemcpyDeviceToHost, d.st), kmcudaMemoryCopyError);
    KMB_CU(cudaStreamSynchronize(d.st), kmcudaRuntimeError);
    total_pairs += p;
  }
  g_prof.mark("knn: exact search of the remainder + copy-out");
  g_prof.report("knn_cuda");
  KMB_INFO("calculated %f of all the distances\n",
           static_cast<double>(total_pairs) / (static_cast<double>(N) * N));  // reference knn.cu:530
  return kmcudaSuccess;
}

}  // namespace kmb
