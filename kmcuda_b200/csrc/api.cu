// api.cu -- the C entry points of include/kmcuda.h and include/kmcuda_b200.h: argument checks, the device list, peer
// access and the k-means copy-out (reference kmcuda.cc:19-137, 402-570); the runs are in job.cu and knn_driver.cu.
#include "job.h"

namespace kmb {

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

namespace {

// which run a k-means request makes
enum class Route { kLloyd, kMinibatch, kBisecting };

// one k-means call, filled by name by each entry point (kmeans_cuda, kmcuda_b200_kmeans_weighted, _relocate,
// _minibatch_init, _restarts, _bisecting and _center_shift); the defaults are those of a plain kmeans_cuda() call
struct KMeansRequest {
  KMCUDAInitMethod init;
  const void* init_params;
  float tolerance;
  float yinyang_t;
  KMCUDADistanceMetric metric;
  uint32_t samples_size;
  uint16_t features_size;
  uint32_t clusters_size;
  uint32_t seed;
  uint32_t device;
  int32_t device_ptrs;
  int32_t fp16x2;
  int32_t verbosity;
  const float* samples;
  const float* weights = nullptr;   // nullptr: the unweighted run
  float* centroids;
  uint32_t* assignments;
  float* average_distance;
  Route route = Route::kLloyd;
  uint32_t batch_size = 0;           // mini-batch
  uint32_t max_steps = 0;            // mini-batch
  uint32_t init_size = 0;            // mini-batch: rows the seeding reads (0 = all, KMCUDA_B200_INIT_SIZE_AUTO)
  bool relocate = false;             // Lloyd / Yinyang
  uint32_t n_init = 1;               // Lloyd / Yinyang, bisecting, mini-batch (with init_size)
  double* inertia = nullptr;         // Lloyd / Yinyang, bisecting
  int32_t strategy = 0;              // bisecting
  uint32_t max_iter = 0;             // bisecting, center shift
  bool center_shift = false;         // scikit-learn's stopping rule with `tol` replaces the reassignment tolerance
  float tol = 0;
  uint32_t* n_iter = nullptr;        // center shift
};

KMCUDAResult kmeans_impl(KMeansRequest r) {
  const int32_t verbosity = r.verbosity;
  KMB_DEBUG("arguments: %d %p %.3f %.2f %d %" PRIu32 " %" PRIu16 " %" PRIu32 " %" PRIu32 " %" PRIu32
            " %d %" PRIi32 " %p %p %p %p\n", r.init, r.init_params, r.tolerance, r.yinyang_t, r.metric,
            r.samples_size, r.features_size, r.clusters_size, r.seed, r.device, r.fp16x2, r.verbosity, r.samples,
            r.centroids, r.assignments, r.average_distance);
  // argument validation: reference check_kmeans_args, kmcuda.cc:19-61
  if (r.clusters_size < 2 || r.clusters_size == UINT32_MAX) return kmcudaInvalidArguments;
  if (r.features_size == 0) return kmcudaInvalidArguments;
  if (r.samples_size < r.clusters_size) return kmcudaInvalidArguments;
  {
    int count = 0;
    cudaGetDeviceCount(&count);
    if (count < 32 && r.device > (1u << count)) return kmcudaNoSuchDevice;
  }
  if (r.samples == nullptr || r.centroids == nullptr || r.assignments == nullptr) return kmcudaInvalidArguments;
  if (!(r.tolerance >= 0 && r.tolerance <= 1)) return kmcudaInvalidArguments;
  if (r.center_shift && !(std::isfinite(r.tol) && r.tol >= 0)) return kmcudaInvalidArguments;
  if (!(r.yinyang_t >= 0 && r.yinyang_t <= 0.5)) return kmcudaInvalidArguments;
  if (static_cast<uint64_t>(r.features_size) * (r.fp16x2 ? 2 : 1) > 65535u) return kmcudaInvalidArguments;
  if (r.init == kmcudaInitMethodKMeansParallel && r.init_params &&
      *static_cast<const uint32_t*>(r.init_params) > kKMeansParallelMaxRounds)
    return kmcudaInvalidArguments;
  if (r.init == kmcudaInitMethodGreedyPlusPlus && r.init_params &&
      *static_cast<const uint32_t*>(r.init_params) > kGreedyPlusPlusMaxTrials)
    return kmcudaInvalidArguments;
  // restarts: at least one run; imported centroids would make every restart the same run
  if (r.n_init == 0 || (r.n_init > 1 && r.init == kmcudaInitMethodImport)) return kmcudaInvalidArguments;
  const char* su = getenv("KMCUDA_B200_STRICT_UPDATE");
  const bool strict = su && su[0] == '1';
  if (r.route == Route::kMinibatch) {
    // one GPU, L2, a real batch; strict mode replays a Lloyd update that mini-batch steps do not have
    if (r.batch_size == 0 || r.metric == kmcudaDistanceMetricCosine || (r.device & (r.device - 1)) != 0 || strict) {
      KMB_INFO("mini-batch k-means takes batch_size >= 1, the L2 metric, one device and no strict update mode\n");
      return kmcudaInvalidArguments;
    }
    // the init stage: an init size of at least K, on a seeding method; several inits only with an init size
    if ((r.init_size != 0 && (r.init == kmcudaInitMethodImport ||
                              (r.init_size != KMCUDA_B200_INIT_SIZE_AUTO && r.init_size < r.clusters_size))) ||
        (r.n_init > 1 && r.init_size == 0)) {
      KMB_INFO("mini-batch k-means takes an init size of at least the number of clusters with a seeding method, and "
               "n_init > 1 only with an init size\n");
      return kmcudaInvalidArguments;
    }
    if (r.device == 0) r.device = 1;
  }
  if (r.route == Route::kBisecting) {
    // one GPU, L2; the 2-means runs start from a random or greedy k-means++ pair; strict mode replays a Lloyd update
    // that bisection does not have
    if (r.metric == kmcudaDistanceMetricCosine || (r.device & (r.device - 1)) != 0 ||
        (r.strategy != 0 && r.strategy != 1) ||
        (r.init != kmcudaInitMethodRandom && r.init != kmcudaInitMethodGreedyPlusPlus) || strict) {
      KMB_INFO("bisecting k-means takes the L2 metric, one device, strategy 0 or 1, the random or greedy k-means++ "
               "init and no strict update mode\n");
      return kmcudaInvalidArguments;
    }
    if (r.device == 0) r.device = 1;
  }
  // strict mode replays the reference's unweighted running sums; there is no weighted reference to replay
  if (r.weights && strict) {
    KMB_INFO("sample weights cannot be combined with KMCUDA_B200_STRICT_UPDATE=1\n");
    return kmcudaInvalidArguments;
  }
  // strict mode replays the reference's update, which leaves empty clusters alone
  if (r.relocate && strict) {
    KMB_INFO("relocating empty clusters cannot be combined with KMCUDA_B200_STRICT_UPDATE=1\n");
    return kmcudaInvalidArguments;
  }
  // strict mode's update keeps a [D][32] centroid tile in shared memory: wider samples would fail after the setup
  if (strict && static_cast<uint64_t>(r.features_size) * (r.fp16x2 ? 2 : 1) > kStrictMaxD) {
    KMB_INFO("KMCUDA_B200_STRICT_UPDATE=1 takes at most %d features\n", kStrictMaxD);
    return kmcudaInvalidArguments;
  }
  if (!r.center_shift)
    KMB_INFO("reassignments threshold: %" PRIu32 "\n", static_cast<uint32_t>(r.tolerance * r.samples_size));
  const uint32_t yy_groups_size = static_cast<uint32_t>(r.yinyang_t * r.clusters_size);
  KMB_DEBUG("yinyang groups: %" PRIu32 "\n", yy_groups_size);
  std::vector<int> dev_ids;
  KMB_RET(list_devices(r.device, verbosity, &dev_ids));
  enable_p2p(dev_ids, r.device_ptrs, verbosity);
  const int m = r.metric == kmcudaDistanceMetricCosine ? 1 : 0;
  const int D = static_cast<int>(r.features_size) * (r.fp16x2 ? 2 : 1);
  const bool fp16x2 = r.fp16x2 != 0;
  g_prof.begin(dev_ids);
  Job job(m, r.samples_size, D, r.clusters_size, verbosity);
  job.weighted = r.weights != nullptr;
  job.relocate_empty = r.relocate;
  job.center_shift = r.center_shift;
  if (r.max_iter) job.max_iter = r.max_iter;
  KMB_RET(job.setup(dev_ids));
  g_prof.mark("setup: exchange (peer / nccl)");
  KMB_RET(job.ingest(r.samples, r.weights, r.device_ptrs, fp16x2));
  g_prof.mark("ingest (H2D / peer copy)");
  if (r.weights) {
    KMB_RET(job.check_weights());
    g_prof.mark("weight check");
  }
  if (r.center_shift) {
    if (r.tol != 0) {   // once per call: every restart stops by the same tolerance
      KMB_RET(job.mean_variance(&job.shift_tol));
      job.shift_tol *= static_cast<double>(r.tol);
    }
    g_prof.mark("center shift tolerance");
    KMB_INFO("center shift tolerance: %.17g, max_iter %" PRIu32 "\n", job.shift_tol, job.max_iter);
  }
  if (verbosity > 1) KMB_RET(print_memory_stats(dev_ids));
  if (r.route == Route::kBisecting) {
    // greedy k-means++: 0 trials = scikit-learn's 2 + floor(ln 2) for the two centres of a bisection
    uint32_t trials = 0;
    if (r.init == kmcudaInitMethodGreedyPlusPlus) {
      trials = r.init_params ? *static_cast<const uint32_t*>(r.init_params) : 0;
      if (trials == 0) trials = greedy_plusplus_trials(2);
    }
    KMB_RET(job.bisecting(r.seed, r.tolerance, r.strategy, r.n_init, trials, r.inertia));
  } else if (r.route == Route::kMinibatch) {
    if (r.init_size == 0) {
      KMB_RET(job.init_centroids(r.init, r.init_params, r.seed, r.device_ptrs, fp16x2, r.centroids));
      g_prof.mark("init centroids");
    } else {
      // scikit-learn's MiniBatchKMeans._check_params_vs_input: 3 b, raised to 3 K, at most N (in 64 bits: 3 b > 2^32)
      const uint64_t b = std::min(r.batch_size, r.samples_size);
      uint64_t m = r.init_size;
      if (r.init_size == KMCUDA_B200_INIT_SIZE_AUTO) {
        m = 3 * b;
        if (m < r.clusters_size) m = 3ull * r.clusters_size;
      }
      m = std::min<uint64_t>(m, r.samples_size);
      KMB_RET(job.minibatch_init(r.init, r.init_params, r.seed, static_cast<uint32_t>(m), r.n_init, r.device_ptrs,
                                 fp16x2));
    }
    KMB_RET(job.minibatch(r.batch_size, r.max_steps, r.tolerance, r.seed));
  } else {
    // under the rule a negative reassignment tolerance: no pass count ends a run or sends Yinyang to Lloyd
    KMB_RET(job.restarts(r.init, r.init_params, r.seed, r.n_init, r.device_ptrs, fp16x2, r.centroids,
                         r.center_shift ? -1.f : r.tolerance, yy_groups_size, r.inertia));
    if (r.n_iter) *r.n_iter = static_cast<uint32_t>(job.n_iter);
  }
  if (r.average_distance) KMB_RET(job.average_distance(r.average_distance));
  g_prof.mark("average distance");
  // copy-out: centroids from the first device (identical everywhere), assignment slices from each shard
  Dev& d0 = job.devs[0];
  KMB_CU(cudaSetDevice(d0.dev), kmcudaRuntimeError);
  KMB_RET(copy_out(r.centroids, d0.C.get(), static_cast<size_t>(r.clusters_size) * D, d0.dev, r.device_ptrs, fp16x2,
                   d0.st, verbosity));
  KMB_CU(cudaStreamSynchronize(d0.st), kmcudaMemoryCopyError);
  for (auto& d : job.devs) {
    KMB_CU(cudaSetDevice(d.dev), kmcudaRuntimeError);
    KMB_RET(copy_out(r.assignments + d.off, d.assign.get(), d.len, d.dev, r.device_ptrs, false, d.st, verbosity));
  }
  KMB_RET(job.sync_all());
  g_prof.mark("copy-out");
  g_prof.report("kmeans_cuda");
  KMB_DEBUG("return kmcudaSuccess\n");
  return kmcudaSuccess;
}

}  // namespace

extern "C" {

KMCUDAResult kmeans_cuda(KMCUDAInitMethod init, const void* init_params, float tolerance,
                         float yinyang_t, KMCUDADistanceMetric metric, uint32_t samples_size,
                         uint16_t features_size, uint32_t clusters_size, uint32_t seed,
                         uint32_t device, int32_t device_ptrs, int32_t fp16x2, int32_t verbosity,
                         const float* samples, float* centroids, uint32_t* assignments,
                         float* average_distance) {
  return kmeans_impl({.init = init, .init_params = init_params, .tolerance = tolerance, .yinyang_t = yinyang_t,
                      .metric = metric, .samples_size = samples_size, .features_size = features_size,
                      .clusters_size = clusters_size, .seed = seed, .device = device, .device_ptrs = device_ptrs,
                      .fp16x2 = fp16x2, .verbosity = verbosity, .samples = samples, .centroids = centroids,
                      .assignments = assignments, .average_distance = average_distance});
}

KMCUDAResult kmcuda_b200_kmeans_weighted(KMCUDAInitMethod init, const void* init_params, float tolerance,
                                         float yinyang_t, KMCUDADistanceMetric metric, uint32_t samples_size,
                                         uint16_t features_size, uint32_t clusters_size, uint32_t seed,
                                         uint32_t device, int32_t device_ptrs, int32_t fp16x2, int32_t verbosity,
                                         const float* samples, const float* weights, float* centroids,
                                         uint32_t* assignments, float* average_distance) {
  return kmeans_impl({.init = init, .init_params = init_params, .tolerance = tolerance, .yinyang_t = yinyang_t,
                      .metric = metric, .samples_size = samples_size, .features_size = features_size,
                      .clusters_size = clusters_size, .seed = seed, .device = device, .device_ptrs = device_ptrs,
                      .fp16x2 = fp16x2, .verbosity = verbosity, .samples = samples, .weights = weights,
                      .centroids = centroids, .assignments = assignments, .average_distance = average_distance});
}

KMCUDAResult kmcuda_b200_kmeans_relocate(KMCUDAInitMethod init, const void* init_params, float tolerance,
                                         float yinyang_t, KMCUDADistanceMetric metric, uint32_t samples_size,
                                         uint16_t features_size, uint32_t clusters_size, uint32_t seed,
                                         uint32_t device, int32_t device_ptrs, int32_t fp16x2, int32_t verbosity,
                                         const float* samples, const float* weights, float* centroids,
                                         uint32_t* assignments, float* average_distance) {
  return kmeans_impl({.init = init, .init_params = init_params, .tolerance = tolerance, .yinyang_t = yinyang_t,
                      .metric = metric, .samples_size = samples_size, .features_size = features_size,
                      .clusters_size = clusters_size, .seed = seed, .device = device, .device_ptrs = device_ptrs,
                      .fp16x2 = fp16x2, .verbosity = verbosity, .samples = samples, .weights = weights,
                      .centroids = centroids, .assignments = assignments, .average_distance = average_distance,
                      .relocate = true});
}

KMCUDAResult kmcuda_b200_kmeans_minibatch(KMCUDAInitMethod init, const void* init_params, float tolerance,
                                          KMCUDADistanceMetric metric, uint32_t samples_size,
                                          uint16_t features_size, uint32_t clusters_size, uint32_t seed,
                                          uint32_t device, int32_t device_ptrs, int32_t fp16x2, int32_t verbosity,
                                          const float* samples, const float* weights, uint32_t batch_size,
                                          uint32_t max_steps, float* centroids, uint32_t* assignments,
                                          float* average_distance) {
  return kmcuda_b200_kmeans_minibatch_init(init, init_params, tolerance, metric, samples_size, features_size,
                                           clusters_size, seed, device, device_ptrs, fp16x2, verbosity, samples,
                                           weights, batch_size, max_steps, 0, 1, centroids, assignments,
                                           average_distance);
}

KMCUDAResult kmcuda_b200_kmeans_minibatch_init(KMCUDAInitMethod init, const void* init_params, float tolerance,
                                               KMCUDADistanceMetric metric, uint32_t samples_size,
                                               uint16_t features_size, uint32_t clusters_size, uint32_t seed,
                                               uint32_t device, int32_t device_ptrs, int32_t fp16x2, int32_t verbosity,
                                               const float* samples, const float* weights, uint32_t batch_size,
                                               uint32_t max_steps, uint32_t init_size, uint32_t n_init,
                                               float* centroids, uint32_t* assignments, float* average_distance) {
  return kmeans_impl({.init = init, .init_params = init_params, .tolerance = tolerance, .yinyang_t = 0.f,
                      .metric = metric, .samples_size = samples_size, .features_size = features_size,
                      .clusters_size = clusters_size, .seed = seed, .device = device, .device_ptrs = device_ptrs,
                      .fp16x2 = fp16x2, .verbosity = verbosity, .samples = samples, .weights = weights,
                      .centroids = centroids, .assignments = assignments, .average_distance = average_distance,
                      .route = Route::kMinibatch, .batch_size = batch_size, .max_steps = max_steps,
                      .init_size = init_size, .n_init = n_init});
}

KMCUDAResult kmcuda_b200_kmeans_restarts(KMCUDAInitMethod init, const void* init_params, float tolerance,
                                         float yinyang_t, KMCUDADistanceMetric metric, uint32_t samples_size,
                                         uint16_t features_size, uint32_t clusters_size, uint32_t seed,
                                         uint32_t device, int32_t device_ptrs, int32_t fp16x2, int32_t verbosity,
                                         const float* samples, const float* weights, int32_t relocate_empty_clusters,
                                         uint32_t n_init, float* centroids, uint32_t* assignments,
                                         float* average_distance, double* inertia) {
  return kmeans_impl({.init = init, .init_params = init_params, .tolerance = tolerance, .yinyang_t = yinyang_t,
                      .metric = metric, .samples_size = samples_size, .features_size = features_size,
                      .clusters_size = clusters_size, .seed = seed, .device = device, .device_ptrs = device_ptrs,
                      .fp16x2 = fp16x2, .verbosity = verbosity, .samples = samples, .weights = weights,
                      .centroids = centroids, .assignments = assignments, .average_distance = average_distance,
                      .relocate = relocate_empty_clusters != 0, .n_init = n_init, .inertia = inertia});
}

KMCUDAResult kmcuda_b200_kmeans_bisecting(KMCUDAInitMethod init, const void* init_params, float tolerance,
                                          KMCUDADistanceMetric metric, uint32_t samples_size,
                                          uint16_t features_size, uint32_t clusters_size, uint32_t seed,
                                          uint32_t device, int32_t device_ptrs, int32_t fp16x2, int32_t verbosity,
                                          const float* samples, const float* weights, int32_t strategy,
                                          uint32_t n_init, uint32_t max_iter, float* centroids,
                                          uint32_t* assignments, float* average_distance, double* inertia) {
  return kmeans_impl({.init = init, .init_params = init_params, .tolerance = tolerance, .yinyang_t = 0.f,
                      .metric = metric, .samples_size = samples_size, .features_size = features_size,
                      .clusters_size = clusters_size, .seed = seed, .device = device, .device_ptrs = device_ptrs,
                      .fp16x2 = fp16x2, .verbosity = verbosity, .samples = samples, .weights = weights,
                      .centroids = centroids, .assignments = assignments, .average_distance = average_distance,
                      .route = Route::kBisecting, .n_init = n_init, .inertia = inertia, .strategy = strategy,
                      .max_iter = max_iter});
}

KMCUDAResult kmcuda_b200_kmeans_center_shift(KMCUDAInitMethod init, const void* init_params, float tol,
                                              float yinyang_t, KMCUDADistanceMetric metric, uint32_t samples_size,
                                              uint16_t features_size, uint32_t clusters_size, uint32_t seed,
                                              uint32_t device, int32_t device_ptrs, int32_t fp16x2, int32_t verbosity,
                                              const float* samples, const float* weights,
                                              int32_t relocate_empty_clusters, uint32_t n_init, uint32_t max_iter,
                                              float* centroids, uint32_t* assignments, float* average_distance,
                                              double* inertia, uint32_t* n_iter) {
  return kmeans_impl({.init = init, .init_params = init_params, .tolerance = 0.f, .yinyang_t = yinyang_t,
                      .metric = metric, .samples_size = samples_size, .features_size = features_size,
                      .clusters_size = clusters_size, .seed = seed, .device = device, .device_ptrs = device_ptrs,
                      .fp16x2 = fp16x2, .verbosity = verbosity, .samples = samples, .weights = weights,
                      .centroids = centroids, .assignments = assignments, .average_distance = average_distance,
                      .relocate = relocate_empty_clusters != 0, .n_init = n_init, .inertia = inertia,
                      .max_iter = max_iter, .center_shift = true, .tol = tol, .n_iter = n_iter});
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
  KMB_RET(knn_run(k, m, samples_size, D, clusters_size, dev_ids, device_ptrs, fp16x2 != 0, verbosity, samples, centroids,
                  assignments, neighbors));
  KMB_DEBUG("return kmcudaSuccess\n");
  return kmcudaSuccess;
}

}  // extern "C"
