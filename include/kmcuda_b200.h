/*
 * kmcuda_b200.h -- shard-level C ABI of the H100-native libKMCUDA (extension, not in the reference).
 *
 * The reference is single-process multi-GPU: one kmeans_cuda() call drives every device in the mask
 * and exchanges results with cudaMemcpyPeerAsync (reference src/private.h:177-183, src/kmeans.cu:
 * 980-990,1014-1024).  A one-process-per-GPU deployment (torch.distributed / MPI ranks) instead
 * owns ONE shard of the samples per rank and needs the hot path as separate steps so that the only
 * collective -- the all-reduce of the per-cluster partial sums -- can be issued by the caller's
 * communicator between them:
 *
 *   kmcuda_b200_assign()        one assignment pass over a device-resident shard
 *                               (reference kernels kmeans_assign_lloyd{,_smallc}, src/kmeans.cu:214-364)
 *   kmcuda_b200_partial_sums()  per-cluster sums + counts of the shard
 *                               (reference kernel kmeans_adjust, src/kmeans.cu:366-423, first half)
 *   kmcuda_b200_finish_update() sums/counts -> centroids after the caller's all-reduce
 *                               (reference METRIC::normalize, src/metric_abstraction.h:138-144,255-272)
 *
 * All pointers are device pointers on the CUDA device that is current when the handle is created;
 * all work is enqueued on `stream` (a cudaStream_t passed as void*; NULL = default stream) and the
 * calls return without synchronising unless stated.  Errors are KMCUDAResult codes.
 */
#ifndef KMCUDA_B200_H
#define KMCUDA_B200_H

#include "kmcuda.h"

#ifdef __cplusplus
extern "C" {
#endif

typedef struct kmcuda_b200_shard kmcuda_b200_shard;

/* Extra KMCUDAInitMethod value accepted by kmeans_cuda() and kmcuda_b200_kmeans_weighted(): k-means|| seeding
 * (Bahmani et al., "Scalable K-Means++", VLDB 2012).  init_params -> uint32_t rounds (NULL or 0 = 5; above 32 is
 * kmcudaInvalidArguments).  c0 is k-means++'s first centroid (srand(seed), rand() % N, redrawn on NaN / zero-weight
 * rows).  Each round draws every row independently with probability 2K w d^2 / sum(w d^2), d = true distance to the
 * nearest candidate so far, through a counter hash of (seed, round, row), so the draws are the same on any number of
 * GPUs; it then runs one assignment pass against that round's candidates.  The candidates, each weighted by the total
 * sample weight nearest to it, are clustered to K by kmcuda_b200_kmeans_weighted(k-means++, tolerance 0.01,
 * yinyang_t 0, same metric and seed) on the first device; with at most K candidates they are the first centroids and
 * random init's walk from srand(seed) fills the rest.  Verbosity >= 1 logs one "k-means|| round" line per round. */
#define kmcudaInitMethodKMeansParallel ((KMCUDAInitMethod)4)

/* kmeans_cuda() with a weight per sample (scikit-learn's sample_weight).  The parameters are those of kmeans_cuda(),
 * plus `weights`: [samples_size] fp32, a host pointer when device_ptrs < 0 and device memory on device `device_ptrs`
 * otherwise (the rule for `samples`; fp32 in fp16x2 mode too).  weights == NULL is the unweighted run.
 * Every weight must be finite and >= 0 and their sum > 0, otherwise kmcudaInvalidArguments; so is a weighted call
 * with KMCUDA_B200_STRICT_UPDATE=1.  The assignment step is unchanged; the centroid update is sum(w x) / sum(w) (L2)
 * or the angular recurrence with weight totals for counts; a cluster whose weight total is 0 is treated as the
 * reference treats an empty cluster (L2: NaN centroid, never chosen again; angular: the same recurrence);
 * k-means++ draws proportionally to w * d, AFK-MC2 uses q = w / 2W + w d^2 / (2 sum w d^2), random init skips rows
 * of weight 0, and average_distance is sum(w d) / sum(w).  With every weight 1 the result is bit-identical to
 * kmeans_cuda(). */
KMCUDAResult kmcuda_b200_kmeans_weighted(KMCUDAInitMethod init, const void *init_params, float tolerance,
                                         float yinyang_t, KMCUDADistanceMetric metric, uint32_t samples_size,
                                         uint16_t features_size, uint32_t clusters_size, uint32_t seed,
                                         uint32_t device, int32_t device_ptrs, int32_t fp16x2, int32_t verbosity,
                                         const float *samples, const float *weights, float *centroids,
                                         uint32_t *assignments, float *average_distance);

/* Creates the per-shard workspace (fp16 centroid table, TMA descriptors, re-check queues, sort
 * buffers) for up to max_samples samples of features_size fp32 features and clusters_size clusters. */
KMCUDAResult kmcuda_b200_shard_create(kmcuda_b200_shard **shard, KMCUDADistanceMetric metric,
                                      uint32_t max_samples, uint16_t features_size,
                                      uint32_t clusters_size, int32_t verbosity);
void kmcuda_b200_shard_destroy(kmcuda_b200_shard *shard);

/* One assignment pass.  samples [n][D] fp32, centroids [K][D] fp32, assignments [n] in/out
 * (0xFFFFFFFF = unassigned), assignments_prev [n] out, *changed (device uint32) += reassignments.
 * Results are bit-identical to the reference's assign kernel on the same inputs. */
KMCUDAResult kmcuda_b200_assign(kmcuda_b200_shard *shard, uint32_t samples_size, const float *samples,
                                const float *centroids, uint32_t *assignments,
                                uint32_t *assignments_prev, uint32_t *changed, void *stream);

/* 1 if the last assign pass ran on the tensor-core (wgmma) filter + exact re-check, 0 if on the exact SIMT
 * kernel; also reports how many samples needed the re-check / the full exact fallback. */
int32_t kmcuda_b200_last_pass_info(kmcuda_b200_shard *shard, uint32_t *rechecked, uint32_t *overflowed);

/* Device time in ms (CUDA events on `stream`) of the tensor-core kernel in the most recent passes,
 * oldest first (up to 64 are kept); returns the number written.  Synchronise the stream first. */
int32_t kmcuda_b200_kernel_times(kmcuda_b200_shard *shard, float *ms_out, int32_t max_out);

/* sums [K][D] fp32 and counts [K] uint32 of the shard (to be all-reduced by the caller). */
KMCUDAResult kmcuda_b200_partial_sums(kmcuda_b200_shard *shard, uint32_t samples_size,
                                      const float *samples, const uint32_t *assignments, float *sums,
                                      uint32_t *counts, void *stream);

/* centroids [K][D] = normalised sums; ccounts [K] = counts.
 * STATEFUL for the angular metric: the reference's incremental update (src/kmeans.cu:366-429) is reproduced as
 * centroid * old count + (member sums now - member sums of the previous call), so the handle remembers the
 * previous member sums.  Call kmcuda_b200_shard_reset() before the first update of every new run (with ccounts
 * zeroed), otherwise the first update of the second run subtracts the last sums of the first. */
KMCUDAResult kmcuda_b200_finish_update(kmcuda_b200_shard *shard, const float *sums,
                                       const uint32_t *counts, float *centroids, uint32_t *ccounts,
                                       void *stream);

/* ---- exchange step of the centroid update for one process per GPU, over peer memory (CUDA IPC; csrc/exchange.cu) ----
 * Replaces the caller's all-reduce between kmcuda_b200_partial_sums() and kmcuda_b200_finish_update() when all ranks
 * sit on GPUs of one node with peer access (NVLink / NVSwitch): every rank reads its peers' partial sums straight from
 * their HBM and adds them in rank order (bit-identical totals on all ranks), one kernel per iteration.  The reference's
 * counterpart is the cudaMemcpyPeerAsync exchange of src/kmeans.cu:980-990,1014-1024 (single process).
 *
 *   create   (every rank; fills handle_out with kmcuda_b200_exchange_handle_bytes() bytes)
 *   all-gather the handles with the caller's communicator (rank-major), then connect
 *   per iteration: buffers -> kmcuda_b200_partial_sums() into them -> reduce -> kmcuda_b200_finish_update() on the totals
 *   destroy  after a barrier of the ranks
 */
typedef struct kmcuda_b200_exchange kmcuda_b200_exchange;
uint32_t kmcuda_b200_exchange_handle_bytes(void);
KMCUDAResult kmcuda_b200_exchange_create(kmcuda_b200_exchange **exchange, uint32_t clusters_size,
                                         uint16_t features_size, int32_t rank, int32_t world, void *handle_out);
KMCUDAResult kmcuda_b200_exchange_connect(kmcuda_b200_exchange *exchange, const void *all_handles);
KMCUDAResult kmcuda_b200_exchange_buffers(kmcuda_b200_exchange *exchange, float **sums, uint32_t **counts);
KMCUDAResult kmcuda_b200_exchange_reduce(kmcuda_b200_exchange *exchange, float *total_sums,
                                         uint32_t *total_counts, void *stream);
/* 0 = clean; non-zero = a peer never arrived within ~20 s (valid after the stream was synchronised) */
uint32_t kmcuda_b200_exchange_error(kmcuda_b200_exchange *exchange);
void kmcuda_b200_exchange_destroy(kmcuda_b200_exchange *exchange);

/* Start of a new clustering run on a reused handle: forgets the cached member sums (see above). */
KMCUDAResult kmcuda_b200_shard_reset(kmcuda_b200_shard *shard, void *stream);

/* Pipeline status of the most recent tensor-core pass, valid after `stream` has been synchronised:
 * 0 = clean; non-zero = a barrier wait inside the kernel timed out (preemption, debugger, a pipeline bug) and
 * the results of that pass must not be used.  kmeans_cuda() / knn_cuda() check this themselves and return
 * kmcudaRuntimeError. */
uint32_t kmcuda_b200_last_error(kmcuda_b200_shard *shard);

/* kmeans_cuda / knn_cuda keep the device memory of their workspace cached between calls (GB-sized cudaMalloc /
 * cudaFree pairs cost more than the kernels of a call); KMCUDA_B200_CACHE_MB caps the amount (default 24576, 0 = no
 * cache).  This returns everything that is cached to the driver. */
void kmcuda_b200_trim_cache(void);

/* Device-memory helpers for language bindings that hand out raw device pointers (the reference's
 * Python binding calls cudaMalloc / cudaMemcpy directly, src/python.cc:298-313,343-352; a ctypes
 * binding cannot reach the statically linked CUDA runtime, so the library re-exports what it needs).
 * direction: 1 = host->device, 2 = device->host, 3 = device->device.  All synchronous. */
KMCUDAResult kmcuda_b200_device_malloc(int32_t device, uint64_t bytes, void **ptr);
KMCUDAResult kmcuda_b200_device_free(int32_t device, void *ptr);
KMCUDAResult kmcuda_b200_device_memcpy(int32_t device, void *dst, const void *src, uint64_t bytes,
                                       int32_t direction);
KMCUDAResult kmcuda_b200_device_synchronize(int32_t device);
int32_t kmcuda_b200_device_count(void);

#ifdef __cplusplus
}
#endif
#endif /* KMCUDA_B200_H */
