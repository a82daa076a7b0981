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

/* Extra KMCUDAInitMethod value accepted by kmeans_cuda(), kmcuda_b200_kmeans_weighted(), _relocate() and _minibatch():
 * greedy k-means++, scikit-learn's k-means++ seeding (sklearn.cluster._kmeans._kmeans_plusplus).  init_params ->
 * uint32_t trials L per round (NULL or 0 = 2 + floor(ln K), scikit-learn's default; 1 = plain d^2 k-means++; above 32
 * is kmcudaInvalidArguments).  c0 is k-means++'s first centroid (srand(seed), rand() % N, redrawn on NaN / zero-weight
 * rows) and d the true distance to it; the mass of a row is m = w d^2 (0 when d is not finite, on rows whose first
 * feature is NaN, on zero-weight rows and on rows already chosen).  Each round r = 1 .. K - 1 draws L trial rows with
 * replacement proportionally to m: trial t is the row of the smallest -ln(u) / m, u a counter hash of (seed, r, t,
 * row), so the trials are the same on any number of GPUs.  The trial whose row lowers the potential sum(m) most (the
 * lowest t on equal potentials, each summed in double in a fixed order) becomes centroid r and d = min(d, distance to
 * it).  When the potential reaches 0 (fewer distinct rows than K), random init's walk from srand(seed) fills the rest
 * with rows not chosen yet.  With every weight 1 the result is bit-identical to the unweighted call.  Verbosity >= 1
 * logs the trial count and the final potential, >= 2 one "greedy k-means++ round" line per round.  With several GPUs
 * the potentials are added in device order, so a pick can differ from one GPU's only where two trials' potentials lie
 * within that rounding. */
#define kmcudaInitMethodGreedyPlusPlus ((KMCUDAInitMethod)5)

/* kmeans_cuda() with a weight per sample (scikit-learn's sample_weight).  The parameters are those of kmeans_cuda(),
 * plus `weights`: [samples_size] fp32, a host pointer when device_ptrs < 0 and device memory on device `device_ptrs`
 * otherwise (the rule for `samples`; fp32 in fp16x2 mode too).  weights == NULL is the unweighted run.
 * Every weight must be finite and >= 0 and their sum > 0, otherwise kmcudaInvalidArguments; so is a weighted call
 * with KMCUDA_B200_STRICT_UPDATE=1.  The assignment step is unchanged; the centroid update is sum(w x) / sum(w) (L2)
 * or the angular recurrence with weight totals for counts; a cluster whose weight total is 0 is treated as the
 * reference treats an empty cluster (L2: NaN centroid, never chosen again; angular: the same recurrence);
 * k-means++ draws proportionally to w * d, AFK-MC2 uses q = w / 2W + w d^2 / (2 sum w d^2) (q = 0, never drawn, on
 * rows of weight 0 and on rows whose distance d to the first centroid is not finite: every row with a NaN feature,
 * which also adds nothing to sum w d^2), random init skips rows of weight 0, and average_distance is
 * sum(w d) / sum(w).  With every weight 1 the result is bit-identical to
 * kmeans_cuda(). */
KMCUDAResult kmcuda_b200_kmeans_weighted(KMCUDAInitMethod init, const void *init_params, float tolerance,
                                         float yinyang_t, KMCUDADistanceMetric metric, uint32_t samples_size,
                                         uint16_t features_size, uint32_t clusters_size, uint32_t seed,
                                         uint32_t device, int32_t device_ptrs, int32_t fp16x2, int32_t verbosity,
                                         const float *samples, const float *weights, float *centroids,
                                         uint32_t *assignments, float *average_distance);

/* kmcuda_b200_kmeans_weighted() (weights == NULL: the unweighted run) that relocates empty clusters, as scikit-learn's
 * KMeans does, instead of the reference's rule.  In every centroid update, after the member sums of all devices are
 * added and before they are normalised, the clusters whose weight total (member count without weights) is 0 are empty;
 * in ascending order they take the rows of a walk over (d desc, row asc), d = a row's exact distance to the centroid it
 * is assigned to (L2: the Kahan sum of squared differences before the square root; angular: the angle).  Rows without a
 * centroid, of weight 0 or with a non-finite d are never taken, nor is a row whose removal would leave its cluster a
 * weight total <= 0 (fp32, in walk order; without weights: its last member).  A taken row x of weight w leaves the
 * donor's sums, count and weight total and becomes the empty cluster's only member: the L2 centroid is w x / w, the
 * angular one x / ||x||.  The assignments are not changed; the next assignment pass moves the rows.  Clusters left
 * empty when the walk runs out keep the reference rule (L2: NaN).  Verbosity >= 1 logs "iteration %d: %u empty
 * clusters relocated" (", %u left empty" when the walk ran out), verbosity >= 2 one line per relocation.  With
 * KMCUDA_B200_STRICT_UPDATE=1 the call returns kmcudaInvalidArguments.  Without empty clusters the result is
 * bit-identical to kmcuda_b200_kmeans_weighted(). */
KMCUDAResult kmcuda_b200_kmeans_relocate(KMCUDAInitMethod init, const void *init_params, float tolerance,
                                         float yinyang_t, KMCUDADistanceMetric metric, uint32_t samples_size,
                                         uint16_t features_size, uint32_t clusters_size, uint32_t seed,
                                         uint32_t device, int32_t device_ptrs, int32_t fp16x2, int32_t verbosity,
                                         const float *samples, const float *weights, float *centroids,
                                         uint32_t *assignments, float *average_distance);

/* Mini-batch k-means (Sculley, "Web-scale k-means clustering", WWW 2010), scikit-learn's MiniBatchKMeans with this
 * library's draws.  init, init_params, tolerance, metric ... weights and the outputs are those of
 * kmcuda_b200_kmeans_weighted(); `init` runs on the full data exactly as there.  Then step s = 1, 2, ... draws
 * b = min(batch_size, samples_size) rows with replacement, row_j = floor(u(seed, s, j) * samples_size) with u a counter
 * hash, assigns them exactly (the reference's argmin), and for every centroid with batch weight W_b > 0 sets
 * c = (c W + S_b) / (W + W_b), W += W_b (W starts at 0; S_b, W_b are the batch's weighted member sums).  Centroids with
 * W < 0.01 max W (at most floor(b / 2) of the smallest) become batch rows drawn proportionally to the weight without
 * replacement, whenever some W is 0 or 10 * clusters_size rows have been drawn since the last time; their W becomes the
 * smallest remaining one.  The run stops after max_steps steps (0 = floor(100 * samples_size / b)), when tolerance > 0
 * and the squared centroid move of a step is <= tolerance * the mean per-feature variance of the samples, or after 10
 * steps without a new minimum of the smoothed batch inertia (step 1 excluded).  One full assignment pass then gives
 * `assignments`.  Verbosity >= 1 logs one "mini-batch step" line per step and the reason it stopped.
 * kmcudaInvalidArguments: batch_size == 0, the cosine metric, a device mask with more than one bit (0 = the first GPU),
 * KMCUDA_B200_STRICT_UPDATE=1.  With every weight 1 the result is bit-identical to weights == NULL. */
KMCUDAResult kmcuda_b200_kmeans_minibatch(KMCUDAInitMethod init, const void *init_params, float tolerance,
                                          KMCUDADistanceMetric metric, uint32_t samples_size, uint16_t features_size,
                                          uint32_t clusters_size, uint32_t seed, uint32_t device, int32_t device_ptrs,
                                          int32_t fp16x2, int32_t verbosity, const float *samples,
                                          const float *weights, uint32_t batch_size, uint32_t max_steps,
                                          float *centroids, uint32_t *assignments, float *average_distance);

/* init_size of kmcuda_b200_kmeans_minibatch_init(): scikit-learn's default, m = 3 b (b = min(batch_size,
 * samples_size)), 3 clusters_size when that is below clusters_size, at most samples_size. */
#define KMCUDA_B200_INIT_SIZE_AUTO 0xFFFFFFFFu

/* Mini-batch k-means with scikit-learn's MiniBatchKMeans init stage (init_size, n_init): kmcuda_b200_kmeans_minibatch()
 * whose seeding reads m = init_size rows instead of all of them, best of n_init inits.  The parameters are those of
 * _minibatch, plus init_size (0 = seed on all rows, which with n_init == 1 is exactly _minibatch;
 * KMCUDA_B200_INIT_SIZE_AUTO = scikit-learn's default above; else m = min(init_size, samples_size)) and n_init.  Init r
 * (r = 0 .. n_init - 1) seeds with seed_r = seed + r * 0x9E3779B9 (mod 2^32), the schedule of _restarts.  When
 * m < samples_size it seeds on the m rows row_j = floor(u * samples_size), u a counter hash of (seed, r, j) with its
 * own tag, drawn with replacement (not by weight), each with its weight: exactly the seeding of a
 * kmcuda_b200_kmeans_weighted() call on those rows with seed_r, for every init method but kmcudaInitMethodImport;
 * otherwise on all rows with seed_r.  With n_init > 1, m validation rows are drawn the same way (their own tag, r = 0),
 * assigned to each init's centroids by the reference's argmin, and the init is ranked by sum w e over them (duplicates
 * included, e the Kahan sum of squared differences, 0 for a row without a centroid); init 0 is the first best and a
 * later one replaces it only with a strictly lower value (NaN never wins).  The mini-batch steps then run from the kept
 * centroids with `seed` exactly as in _minibatch.  Verbosity >= 1 with init_size != 0 adds, after each seeding's own
 * lines, "mini-batch init r/n_init: seed s, m rows" (r from 1), with ", validation inertia %.17g" when n_init > 1, and
 * then "mini-batch init: kept init r/n_init".  kmcudaInvalidArguments: what _minibatch rejects, n_init == 0, n_init > 1
 * with init_size == 0, init_size != 0 with kmcudaInitMethodImport, an init_size below clusters_size other than 0 and
 * KMCUDA_B200_INIT_SIZE_AUTO, and sampled rows whose weights sum to 0. */
KMCUDAResult kmcuda_b200_kmeans_minibatch_init(KMCUDAInitMethod init, const void *init_params, float tolerance,
                                               KMCUDADistanceMetric metric, uint32_t samples_size,
                                               uint16_t features_size, uint32_t clusters_size, uint32_t seed,
                                               uint32_t device, int32_t device_ptrs, int32_t fp16x2, int32_t verbosity,
                                               const float *samples, const float *weights, uint32_t batch_size,
                                               uint32_t max_steps, uint32_t init_size, uint32_t n_init,
                                               float *centroids, uint32_t *assignments, float *average_distance);

/* k-means restarts, scikit-learn's KMeans(n_init=...): n_init seedings and runs over one ingest of the samples, keeping
 * the run of lowest inertia.  The parameters up to `weights` are those of kmcuda_b200_kmeans_relocate(); restart r
 * (r = 0 .. n_init - 1) is exactly what one kmcuda_b200_kmeans_relocate() call (relocate_empty_clusters != 0) or one
 * kmcuda_b200_kmeans_weighted() call (relocate_empty_clusters == 0) runs with seed_r = seed + r * 0x9E3779B9 (mod 2^32):
 * the seeding, then the Lloyd or Yinyang run.  The samples are ingested and the weights checked once per call.
 * The inertia of a run is sum_i w_i e_i over all rows (w_i = 1 without weights): L2 e_i = the Kahan sum of squared
 * differences to the row's centroid, angular e_i = the angle to it, squared; a row without a centroid or with a
 * non-finite e_i adds 0.  Each device adds its block partials in double in a fixed order, the host adds the devices in
 * device order.  Restart 0 is the first best; a later restart replaces it only with a strictly lower inertia (ties keep
 * the earlier one, NaN never wins), so with several GPUs the pick can differ from one GPU's only where two inertias lie
 * within the rounding of that sum.  The outputs are the kept restart's centroids and assignments; average_distance (if
 * not NULL) is computed on that restart, and *inertia (if not NULL) is its inertia against the fp32 centroids (before
 * any fp16x2 narrowing of the copy-out).  With n_init == 1 the centroids, assignments, average distance and log are
 * bit-identical to the corresponding kmcuda_b200_kmeans_relocate() / _weighted() / kmeans_cuda() call; only *inertia
 * is added.  kmcudaInvalidArguments: n_init == 0, or n_init > 1 with kmcudaInitMethodImport (every restart would be the
 * same run).  Verbosity >= 1 with n_init > 1 logs each restart's own lines in turn, "restart r/n_init: seed s, inertia
 * %.17g" after restart r, and "restarts: kept restart r, inertia %.17g" at the end. */
KMCUDAResult kmcuda_b200_kmeans_restarts(KMCUDAInitMethod init, const void *init_params, float tolerance,
                                         float yinyang_t, KMCUDADistanceMetric metric, uint32_t samples_size,
                                         uint16_t features_size, uint32_t clusters_size, uint32_t seed,
                                         uint32_t device, int32_t device_ptrs, int32_t fp16x2, int32_t verbosity,
                                         const float *samples, const float *weights /* NULL = unweighted */,
                                         int32_t relocate_empty_clusters, uint32_t n_init,
                                         float *centroids, uint32_t *assignments, float *average_distance,
                                         double *inertia /* NULL = not wanted */);

/* k-means with scikit-learn's stopping rule, KMeans(tol=..., max_iter=...): kmcuda_b200_kmeans_restarts() with the
 * reassignment `tolerance` replaced by the centre-shift `tol`, plus max_iter (0 = 300) and *n_iter.  It accepts what
 * _restarts accepts and rejects what it rejects, and in addition a negative or non-finite tol.  The rule (DESIGN.md §4p):
 *   tol_abs = tol * mean_f Var(X_f), the unweighted population variance of every feature in double (scikit-learn's
 *     _tolerance), computed once per call; tol == 0 gives 0 without the variance pass.  With a non-finite sample tol_abs
 *     is not finite and only equal labels or max_iter can stop a run.
 *   Iteration i = 1, 2, ... is one assignment pass (pass i), the centroid update (with relocation if asked for), then
 *     S_i = sum_c ||c_new - c_old||^2 in double in a fixed order; a centroid whose old or new coordinates are not finite
 *     (a cluster that died under the reference's empty-cluster rule) adds 0.
 *   The run stops when pass i (i > 1) makes no reassignment ("equal labels": its labels and the centroids they were
 *     made against stand, n_iter = i); when S_i <= tol_abs ("tolerance") or i == max_iter ("max_iter"): pass i + 1 is
 *     the final E step and n_iter = i.  The shift or the cap at i wins over equal labels at pass i + 1, as in
 *     scikit-learn's _kmeans_single_lloyd.
 * S_i is read back with pass i + 1's reassignment count, so an iteration keeps its one host round trip.  Yinyang runs
 * make the same decisions at the same points; its Lloyd draft and the adaptive switch back to Lloyd are unchanged.
 * Every restart runs this rule; *inertia is taken after the final E step and *n_iter (if not NULL) is the kept
 * restart's.  tol == 0 with a large enough max_iter stops where _restarts(tolerance = 0) stops, with the same results.
 * Log: the "iteration %d: %u reassignments" lines are those of every pass (the final E step is pass n_iter + 1), the
 * "reassignments threshold" line becomes "center shift tolerance: %.17g, max_iter %u", verbosity >= 1 adds "stopped
 * at iteration %d: <equal labels | tolerance | max_iter>" and verbosity >= 2 "center shift %d: %.17g (tolerance %.17g)"
 * per update. */
KMCUDAResult kmcuda_b200_kmeans_center_shift(KMCUDAInitMethod init, const void *init_params, float tol,
                                             float yinyang_t, KMCUDADistanceMetric metric, uint32_t samples_size,
                                             uint16_t features_size, uint32_t clusters_size, uint32_t seed,
                                             uint32_t device, int32_t device_ptrs, int32_t fp16x2, int32_t verbosity,
                                             const float *samples, const float *weights /* NULL = unweighted */,
                                             int32_t relocate_empty_clusters, uint32_t n_init,
                                             uint32_t max_iter /* 0 = 300 */, float *centroids,
                                             uint32_t *assignments, float *average_distance,
                                             double *inertia /* NULL = not wanted */,
                                             uint32_t *n_iter /* NULL = not wanted */);

/* Bisecting k-means, scikit-learn's BisectingKMeans: the K clusters are made by splitting one cluster in two at a time
 * with a 2-means run inside it, on one GPU (device: a mask of at most one bit, 0 = the first GPU), L2 only.  The
 * parameters up to `weights` are those of kmcuda_b200_kmeans_minibatch().  strategy 0 splits the leaf of largest
 * inertia sum w e, strategy 1 the leaf of most rows (scikit-learn's bisecting_strategy "biggest_inertia" and
 * "largest_cluster"); equal scores take the leaf that comes first in the tree's depth-first, left-first order, which
 * is also the order of the output clusters.  Each bisection runs n_init inits (kmcudaInitMethodRandom: the two rows of
 * positive weight of smallest -ln(u) / w; kmcudaInitMethodGreedyPlusPlus, init_params a uint32_t number of trials L,
 * 0 or NULL = 2: centre 0 the row of smallest -ln(u) / w, centre 1 the best of L d^2-sampled trial rows by the
 * potential they leave, greedy k-means++ restricted to the node) with at most max_iter (0 = 300) Lloyd iterations, and
 * keeps the first init
 * whose inertia no later one beats by more than a factor 1 - 1e-6.  A 2-means run stops when its labels repeat or when
 * sum ||dc||^2 <= tolerance * (the mean of the unweighted per-feature variances of the samples), scikit-learn's KMeans
 * scaling (BisectingKMeans passes its tol unscaled).  A child left without weight takes the farthest row of positive
 * weight of the other child.  The draws depend on (seed, node, init) only and every double total is added in a fixed
 * order, so the result depends on no launch shape; with every weight 1 it is bit-identical to weights == NULL.
 * *inertia (if not NULL) is sum w ||x - c||^2 of the result, average_distance as for kmeans_cuda().  Verbosity >= 1 logs
 * one "bisecting: split" line per split in pick order and a final line with the waves, the nodes bisected and the
 * inertia; verbosity >= 2 one line per (node, init) with its iterations, stop reason and inertia.
 * kmcudaInvalidArguments: the cosine metric, more than one device, strategy not 0 or 1, n_init == 0, an init other
 * than kmcudaInitMethodRandom or kmcudaInitMethodGreedyPlusPlus (at most 32 trials), KMCUDA_B200_STRICT_UPDATE=1, a
 * non-finite sample, data from which fewer than K clusters can be made (too few distinct rows of positive weight), an
 * n_init * K too large for the 32-bit segment indices, and everything kmeans_cuda() rejects. */
KMCUDAResult kmcuda_b200_kmeans_bisecting(KMCUDAInitMethod init, const void *init_params, float tolerance,
                                          KMCUDADistanceMetric metric, uint32_t samples_size, uint16_t features_size,
                                          uint32_t clusters_size, uint32_t seed, uint32_t device, int32_t device_ptrs,
                                          int32_t fp16x2, int32_t verbosity, const float *samples,
                                          const float *weights /* NULL = unweighted */,
                                          int32_t strategy /* 0 = biggest inertia, 1 = largest cluster */,
                                          uint32_t n_init, uint32_t max_iter /* 0 = 300 */, float *centroids,
                                          uint32_t *assignments, float *average_distance,
                                          double *inertia /* NULL = not wanted */);

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
