// job.h -- host side of a call: per-device state, the k-means Job (job.cu, seeding.cu), copy routes (transfer.cu), k-NN.
#pragma once
#include <nccl.h>  // types only: NCCL is bound at run time (job.cu)

#include <algorithm>
#include <chrono>
#include <cinttypes>
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <initializer_list>
#include <memory>
#include <string>
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
static const uint32_t kGreedyPlusPlusMaxTrials = 32;    // greedy k-means++ trials per round (kGppMaxTrials)
// greedy k-means++ trials per round when init_params gives none: scikit-learn's 2 + floor(ln k) for k centres
inline uint32_t greedy_plusplus_trials(uint32_t k) {
  return 2 + static_cast<uint32_t>(std::log(static_cast<double>(k)));
}

// Device teardown (transfer.cu).  A buffer goes back to the pool only after its stream has been synchronised
// (kernels.h), also when a call returns early on an error while work is still queued: the owner of several devices
// syncs all their streams first (a device's stream may read its peers' buffers), then each device retires its stream
// (synchronise, destroy the events and the stream) before its buffers are released.
void sync_stream(int dev, cudaStream_t st);
void retire_stream(int dev, cudaStream_t st, std::initializer_list<cudaEvent_t> events);

// one device's share of a k-means job; owns its stream and events (constructed in place, never copied or moved)
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
  // relocation of empty clusters (Job::relocate; allocated at the first update that has an empty cluster): the row keys
  // of this shard, the top-T selection's scratch, and the relocated rows with their (cluster, donor, weight) records
  DevBuf<uint64_t> rl_keys, rl_state, rl_sel, rl_top;
  DevBuf<uint32_t> rl_hist, rl_nsel, rl_meta, rl_idx;
  DevBuf<float> rl_x;
  DevBuf<char> rl_tmp;
  uint32_t rl_cap = 0;
  // scikit-learn's stopping rule (Job::center_shift): the centroids before a Lloyd update and the per-centroid squared
  // moves (first device only), and the centre shift S read back with the next pass (every device, read from the first)
  DevBuf<float> Cold;
  DevBuf<double> dsq, d_shift;
  cudaEvent_t ev_partial = nullptr;   // this device's partial sums are complete
  cudaEvent_t ev_reduced = nullptr;   // this device has finished reading every peer's partial sums
  ncclComm_t comm = nullptr;          // owned by the per-process cache (Job::setup)

  Dev() = default;
  Dev(const Dev&) = delete;
  Dev& operator=(const Dev&) = delete;
  ~Dev() {
    retire_stream(dev, st, {ev_partial, ev_reduced});
    shard.reset();
  }
};

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
extern PhaseProfile g_prof;   // the library is not re-entrant (kmcuda.h:25-26), one profile is enough (job.cu)

// Copy routes (transfer.cu) on device `dev` (current) and stream `st`.  The caller's pointers are host memory when
// device_ptrs < 0, else memory of device `device_ptrs`.  Failures: allocation -> kmcudaMemoryAllocationFailure, copy or
// synchronisation -> kmcudaMemoryCopyError, fp16 conversion launch -> kmcudaRuntimeError.
// In: `count` elements at `src` into `dst`, borrowed when `src` lives on `dev`, needs no widening and `borrow` allows it
// (read-only uses), else allocated and filled from the host (staged pageable copy when `staged`) or a peer.  fp16x2
// (floats only): `src` holds halves, widened through a temporary synchronised before it dies (read in place if borrowable).
template <typename T>
KMCUDAResult copy_in(DevBuf<T>& dst, const T* src, size_t count, int dev, int device_ptrs, bool fp16x2, cudaStream_t st,
                     int verbosity, bool borrow = true, bool staged = true);
// Out: `count` elements of `src` to the caller's `dst`, enqueued; fp16x2: narrowed through a synchronised temporary.
template <typename T>
KMCUDAResult copy_out(T* dst, const T* src, size_t count, int dev, int device_ptrs, bool fp16x2, cudaStream_t st,
                      int verbosity);

class Job {
 public:
  Job(int metric, uint32_t N, int D, uint32_t K, int verbosity)
      : metric(metric), N(N), D(D), K(K), verbosity(verbosity) {}
  ~Job() { drain(); }

  const int metric;
  const uint32_t N;
  const int D;
  const uint32_t K;
  const int verbosity;
  std::vector<Dev> devs;        // sized once by setup()
  bool peer_exchange = false;   // multi-GPU update through peer memory (NVLink / NVSwitch) instead of NCCL
  bool weighted = false;        // per-sample weights (kmcuda_b200_kmeans_weighted); set before setup()
  bool relocate_empty = false;  // relocate empty clusters in update() (kmcuda_b200_kmeans_relocate)
  // scikit-learn's stopping rule instead of the reference's (kmcuda_b200_kmeans_center_shift, DESIGN.md §4p); set before
  // setup().  The runs are then given a negative reassignment tolerance, which never stops them.
  bool center_shift = false;
  double shift_tol = 0;         // tol times the mean per-feature variance (mean_variance)
  uint32_t max_iter = 300;      // the last update of a run (of a 2-means run in bisecting())
  int n_iter = 0;               // iterations of the last run (of the kept restart after restarts()), 0 while it runs
  uint32_t relocated = 0;       // rows relocated by the last relocate(), still in every device's rl_x / rl_meta
  double wtotal = 0;            // sum of the weights (check_weights)
  std::vector<float> host_w;    // host copy of the weights for the host-side seeding steps (load_host_weights)

  KMCUDAResult setup(const std::vector<int>& dev_ids);
  KMCUDAResult ingest(const float* samples, const float* weights, int device_ptrs, bool fp16x2);
  KMCUDAResult check_weights();
  KMCUDAResult load_host_weights();
  KMCUDAResult sync_all();
  void drain() {   // synchronises every device's stream (teardown: errors are not reported)
    for (auto& d : devs) sync_stream(d.dev, d.st);
  }
  // declared after a function's own device buffers: they go back to the pool only after every stream has drained
  struct Drain {
    Job& job;
    ~Drain() { job.drain(); }
  };
  // One round trip per device: for each (src, out) pair, the scalar *src(i) of device i is copied back on its stream
  // into (*out)[i], then the stream is synchronised.  The values are in device order, so that callers add them in it.
  template <typename... Reads>
  KMCUDAResult gather(Reads... reads) {
    for (size_t i = 0; i < devs.size(); i++) {
      KMB_CU(cudaSetDevice(devs[i].dev), kmcudaRuntimeError);
      KMB_CU(read_back(i, reads...), kmcudaMemoryCopyError);
      KMB_CU(cudaStreamSynchronize(devs[i].st), kmcudaRuntimeError);
    }
    return kmcudaSuccess;
  }
  template <typename F, typename T, typename... More>
  cudaError_t read_back(size_t i, F src, std::vector<T>* out, More... more) {
    out->resize(devs.size());
    cudaError_t e = cudaMemcpyAsync(&(*out)[i], src(i), sizeof(T), cudaMemcpyDeviceToHost, devs[i].st);
    if constexpr (sizeof...(More) > 0)
      if (e == cudaSuccess) e = read_back(i, more...);
    return e;
  }
  KMCUDAResult set_centroids_from_host(const float* hostC);
  KMCUDAResult fetch_row(uint32_t idx, float* host_row);
  KMCUDAResult init_centroids(KMCUDAInitMethod method, const void* init_params, uint32_t seed,
                              int device_ptrs, bool fp16x2, const float* user_centroids);
  KMCUDAResult draw_first_centroid(float* hostC, uint32_t* first_out);
  KMCUDAResult fill_random(float* hostC, uint32_t start, const std::vector<char>* taken, const char* what);
  KMCUDAResult init_random();
  KMCUDAResult init_plusplus();
  KMCUDAResult init_afkmc2(uint32_t m, uint32_t seed);
  KMCUDAResult init_kmeans_parallel(uint32_t rounds, uint32_t seed);
  KMCUDAResult init_greedy_plusplus(uint32_t trials, uint32_t seed);
  // *shift (with the rule): the centre shift of the update before this pass, read back in the same round trip
  KMCUDAResult assign_pass(uint32_t* changed, double* shift = nullptr);
  KMCUDAResult update(int iter);
  KMCUDAResult lloyd_update(int iter);
  KMCUDAResult shift_of(const float* Cold);
  // scikit-learn's _tolerance before its factor tol: the mean over the features of their population variances
  KMCUDAResult mean_variance(double* out);
  bool shift_stop(int iter, uint32_t changed, double shift);
  KMCUDAResult relocate(int iter);
  // iter == 0: a fresh run; iter > 0: the run continues after pass `iter` (Job::yinyang)
  KMCUDAResult lloyd(float tolerance, int iter = 0, int* iter_out = nullptr, uint32_t* changed_out = nullptr);
  KMCUDAResult yinyang(float tolerance, uint32_t G);
  KMCUDAResult minibatch(uint32_t batch_size, uint64_t max_steps, float tolerance, uint32_t seed);
  // the init stage of a mini-batch run (DESIGN.md §4q) on the first device: n_init seedings, init r on m rows drawn
  // with seed_r (all rows when m >= N), the one of lowest inertia on m validation rows left in C
  KMCUDAResult minibatch_init(KMCUDAInitMethod method, const void* init_params, uint32_t seed, uint32_t m,
                              uint32_t n_init, int device_ptrs, bool fp16x2);
  double lloyd_iter_ms = 0;   // wall time of the fastest complete Lloyd iteration of this run (assign pass + update), 0 = none yet
  KMCUDAResult group_centroids(uint32_t G, std::vector<uint32_t>* groups);
  // n_init seedings + Lloyd / Yinyang runs, the one of lowest inertia left in C / assign (kmcuda_b200_kmeans_restarts);
  // n_init == 1 and inertia_out == nullptr is the plain run
  KMCUDAResult restarts(KMCUDAInitMethod method, const void* init_params, uint32_t seed, uint32_t n_init,
                        int device_ptrs, bool fp16x2, const float* user_centroids, float tolerance, uint32_t G,
                        double* inertia_out);
  // bisecting k-means (kmcuda_b200_kmeans_bisecting, DESIGN.md §4o) on the first device: C / assign, *inertia_out;
  // trials = 0: random init, else greedy k-means++ with that many trials
  KMCUDAResult bisecting(uint32_t seed, float tolerance, int strategy, uint32_t n_init, uint32_t trials,
                         double* inertia_out);
  KMCUDAResult inertia(double* out);
  KMCUDAResult average_distance(float* out);
};

// knn_cuda() after argument checks on the devices `dev_ids` (peer access enabled): knn_driver.cu
KMCUDAResult knn_run(uint16_t k, int metric, uint32_t N, int D, uint32_t K, const std::vector<int>& dev_ids,
                     int32_t device_ptrs, bool fp16x2, int verbosity, const float* samples, const float* centroids,
                     const uint32_t* assignments, uint32_t* neighbors);

}  // namespace kmb
