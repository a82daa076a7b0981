// kernels.h -- host-callable launchers of the device code (one CUDA stream per device context).
//
// Two families:
//   * exact kernels (simt_kernels.cu, knn_kernels.cu): bit-for-bit the reference's fp32 arithmetic
//     (exact.cuh); they make every decision that leaves the library.
//   * the tensor-core filter (assign_tc.cu): wgmma fp16 distance GEMM that proposes, per sample,
//     the short list of centroids the exact re-check has to look at.
#pragma once
#include <cuda_runtime.h>
#include <cstdint>
#include <vector>

namespace kmb {

inline unsigned cdiv(size_t a, size_t b) { return static_cast<unsigned>((a + b - 1) / b); }

// Device-memory cache (shard.cu).  kmeans_cuda / knn_cuda allocate their whole workspace at entry like the reference
// (wrappers.h:16-21); GB-sized cudaMalloc / cudaFree pairs can cost a call more than its kernels, so freed blocks
// are kept per device and handed to the next call.  Blocks are
// only returned here after the owning stream has been synchronised.  KMCUDA_B200_CACHE_MB caps what is kept (default
// 24576; 0 disables the cache); kmcuda_b200_trim_cache() releases everything.
cudaError_t pool_alloc(void** p, size_t bytes);   // on the current device
void pool_free(void* p);
void pool_trim();

constexpr uint32_t kUntouched = 0xFFFFFFFEu;  // "no centroid won": leave the assignment alone
constexpr uint32_t kOverflowRow = 0xFFFFFFFDu;  // row-list pass: this position waits for the exact list pass

// The one-CTA-per-row exact kernels (exact_rows_few_kernel, yy_rows_cta_kernel) stage the sample row in shared memory
// up to this many features (64 KB, past the 48 KB a launch gets without opting in) and read longer rows from global
// memory, where every thread of the CTA loads the same address at each step.  The arithmetic is the same either way.
constexpr int kRowStageMaxD = 16384;

// ---- exact Lloyd assignment (all K centroids), optional row list -------------------------------
// result[i] = argmin (strict <, ascending index), K for "insane" rows, kUntouched if nothing wins.
// rows == nullptr: rows 0..n-1; else the n row ids in rows[] (device), results still indexed by row.
cudaError_t launch_csqr(int metric, const float* C, uint32_t K, int D, float* csq, cudaStream_t st);
cudaError_t launch_assign_exact(int metric, const float* X, const float* C, const float* csq,
                                uint32_t n, int D, uint32_t K, const uint32_t* rows,
                                const uint32_t* d_nrows, uint32_t* result, cudaStream_t st);

// prev[i]=assign[i]; assign[i]=result[i] unless kUntouched; *changed += #(assign changed)
cudaError_t launch_finalize_assign(uint32_t n, const uint32_t* result, uint32_t* assign,
                                   uint32_t* prev, uint32_t* d_changed, cudaStream_t st);

// ---- centroid update ----------------------------------------------------------------------------
// Deterministic: stable radix sort of (assignment, index), then per-cluster Kahan sums in index order.
struct UpdateWorkspace {
  uint32_t *keys_in = nullptr, *keys_out = nullptr, *vals_in = nullptr, *vals_out = nullptr;
  uint32_t* offsets = nullptr;   // [K+1]
  float* partial = nullptr;      // [update_partial_rows(max_n, K)][D]: one row per (chunk, cluster) run
  float* partial_w = nullptr;    // [update_partial_rows(max_n, K)]: weight total per run (weighted update only)
  void* cub_tmp = nullptr;
  size_t cub_tmp_bytes = 0;
  uint32_t iota_n = 0;           // vals_in[0 .. iota_n) already holds the identity permutation
};
#ifndef KMB_SUM_CHUNK
#define KMB_SUM_CHUNK 512
#endif
constexpr uint32_t kSumChunk = KMB_SUM_CHUNK;   // sorted positions per CTA of the member-sum kernel
size_t update_partial_rows(uint32_t n, uint32_t K);
size_t update_cub_bytes(uint32_t n);
// sums[K][D] (fp32) and counts[K] (uint32) of this shard's samples.  With sample weights w[n]: sums = sum of w_i x_i
// and wsums[K] = sum of w_i over the members (ws.partial_w must be set); counts stay member counts.
// vals (optional, [n]): the sample row of each entry (mini-batch: entries are sampled rows, w is indexed by row);
// nullptr = entry i is row i
cudaError_t launch_partial_sums(const float* X, uint32_t n, int D, uint32_t K, const uint32_t* assign,
                                UpdateWorkspace& ws, float* sums, uint32_t* counts, cudaStream_t st,
                                const float* w = nullptr, float* wsums = nullptr, const uint32_t* vals = nullptr);
// strict parity mode: the reference's running-sum update replayed in sample order (simt_kernels.cu).  Each 32-thread
// CTA keeps its centroids as a [D][32] tile in at most 200 KB of shared memory, hence the feature limit.
constexpr int kStrictMaxD = 200 * 1024 / (32 * sizeof(float));   // 1600
size_t strict_update_cub_bytes(uint32_t n);
cudaError_t launch_strict_update(int metric, const float* X, uint32_t n, int D, uint32_t K, const uint32_t* prev,
                                 const uint32_t* cur, float* C, uint32_t* ccounts, uint32_t* keys_in,
                                 uint32_t* vals_in, uint32_t* keys_out, uint32_t* vals_out, uint32_t* offsets,
                                 void* cub_tmp, size_t cub_bytes, cudaStream_t st);
// multi-GPU exchange through peer memory: out_sums = sums[0] + sums[1] + ... (device order, so every GPU computes
// the same bits), out_counts likewise; the pointers may live on other GPUs (peer access enabled by the caller)
constexpr int kMaxPeers = 32;
struct PeerBuffers {
  int n;
  const float* sums[kMaxPeers];
  const uint32_t* counts[kMaxPeers];
};
cudaError_t launch_peer_reduce(const PeerBuffers& pb, uint32_t K, int D, float* out_sums, uint32_t* out_counts,
                               cudaStream_t st);
// weighted update: out = p[0] + p[1] + ... (device order) of `count` floats, the per-cluster weight totals
struct PeerF32 {
  int n;
  const float* p[kMaxPeers];
};
cudaError_t launch_peer_sum_f32(const PeerF32& pb, size_t count, float* out, cudaStream_t st);
// C = sums/count (L2, NaN for empty) or sums/||sums|| (cosine); ccounts = counts.  Weighted (wsums != nullptr): the
// count is replaced by the weight total, cweights[K] holds it between updates (the cosine recurrence's old count)
cudaError_t launch_normalize(int metric, const float* sums, const uint32_t* counts, uint32_t K, int D,
                             float* C, uint32_t* ccounts, float* prev_sums, cudaStream_t st,
                             const float* wsums = nullptr, float* cweights = nullptr);
// sample weights: flags[0] |= 1 if some w is NaN, infinite or negative; *total += sum of w (both zeroed by the caller)
cudaError_t launch_check_weights(const float* w, uint32_t n, uint32_t* flags, double* total, cudaStream_t st);

// ---- Yinyang -------------------------------------------------------------------------------------
// bounds layout [n][G+1] (one contiguous record per sample): [0] = upper bound, [1+g] = lower bound of group g
cudaError_t launch_yy_init(int metric, const float* X, const float* C, uint32_t n, int D, uint32_t K,
                           uint32_t G, const uint32_t* assign, const uint32_t* groups, float* bounds,
                           cudaStream_t st);
// exact refresh of the listed rows only (rows[0 .. *d_nrows))
cudaError_t launch_yy_init_rows(int metric, const float* X, const float* C, uint32_t n, int D, uint32_t K,
                                uint32_t G, const uint32_t* assign, const uint32_t* groups, float* bounds,
                                const uint32_t* rows, const uint32_t* d_nrows, cudaStream_t st);
cudaError_t launch_yy_drifts(int metric, const float* Cnew, const float* Cold, uint32_t K, int D,
                             uint32_t G, const uint32_t* groups, float* drift, float* maxdrift,
                             cudaStream_t st);
struct TcPlan;
// one Yinyang iteration after the centroid update (yinyang.cu): bound decay + group filter, exact tightening of
// the upper bound, tensor-core candidate pass over the surviving rows, bound / assignment update
struct YyWorkspace {
  float* minlb;            // [n]
  uint32_t* tight_rows;    // [n]
  uint32_t* tight_cand;    // [n]
  float* tight_score;      // [n]
  uint32_t* passed;        // [n]
  uint32_t* gsize;         // [G] members per group (NaN centroids excluded)
  uint32_t* counters;      // [4]: tight, passed, (spare)
};
cudaError_t launch_yy_group_sizes(const uint32_t* groups, uint32_t K, uint32_t G, uint32_t* gsize, cudaStream_t st);
cudaError_t launch_yy_step(int metric, TcPlan* plan, const float* X, const float* C, const float* csq, uint32_t n,
                           int D, uint32_t K, uint32_t G, const uint32_t* groups, const float* drift,
                           const float* maxdrift, uint32_t* assign, uint32_t* prev, float* bounds,
                           const YyWorkspace& ws, uint32_t* d_changed, bool reference_order_scan, cudaStream_t st);

// ---- misc ------------------------------------------------------------------------------------------
// w (sample weights, optional): *d_sum accumulates w_i * d_i
cudaError_t launch_average_distance(int metric, const float* X, const float* C, uint32_t n, int D,
                                    const uint32_t* assign, double* d_sum, cudaStream_t st, const float* w = nullptr);
cudaError_t launch_afkmc2_min_dist(int metric, const float* X, const float* C, int D, uint32_t k,
                                   const uint32_t* rows, uint32_t m, float* min_dists, cudaStream_t st);
// w (optional): dists[] stays the plain minimum distance, *d_sum accumulates w_i * d_i; rows whose first feature is NaN
// get the distance nan_row_dist (AFK-MC2 passes NaN to tell them from rows at distance 0)
cudaError_t launch_plusplus_step(int metric, const float* X, uint32_t n, int D, const float* centroid,
                                 int first, float* dists, double* d_sum, cudaStream_t st, const float* w = nullptr,
                                 float nan_row_dist = 0.f);
// device-resident k-means++ round (simt_kernels.cu): bsum / bpre hold ceil(n / 256) + 1 doubles, chosen [K];
// w (optional): the draw is proportional to w_i * d_i and never picks a zero-weight row
cudaError_t launch_plusplus_round(int metric, const float* X, uint32_t n, int D, float* C, uint32_t i, double choice,
                                  float* dists, double* bsum, double* bpre, uint32_t* chosen, cudaStream_t st,
                                  const float* w = nullptr);
// ---- k-means|| seeding (kmeans_parallel.cu) -------------------------------------------------------------------------
// running-minimum update of a round: assign == nullptr is the start (every row against cand[0] = c0, nearest = 0),
// otherwise row i compares its true distance to cand[assign[i]] (assign[i] < ncand) with dists[i] and on e < d takes
// nearest[i] = base + assign[i].  bsum[kmp_blocks(n)] receives the per-block partials of sum w_i d_i^2 (w optional).
uint32_t kmp_blocks(uint32_t n);
cudaError_t launch_kmp_update(int metric, const float* X, uint32_t n, int D, const float* cand, uint32_t ncand,
                              const uint32_t* assign, uint32_t base, float* dists, uint32_t* nearest, const float* w,
                              double* bsum, cudaStream_t st);
// the draw of round `round`: flags[i] = u(seed, round, off + i) < ell * w_i d_i^2 / phi; idx[0 .. *d_count) = the
// drawn local row ids, ascending.  tmp: kmp_select_bytes(n) bytes
size_t kmp_select_bytes(uint32_t n);
cudaError_t launch_kmp_draw(const float* dists, const float* w, uint32_t n, uint32_t off, uint32_t seed, uint32_t round,
                            double ell, double phi, uint8_t* flags, uint32_t* idx, uint32_t* d_count, void* tmp,
                            size_t tmp_bytes, cudaStream_t st);
// out[j][:] = X[idx[j]][:]
cudaError_t launch_kmp_gather(const float* X, int D, const uint32_t* idx, uint32_t cnt, float* out, cudaStream_t st);
// candidate weights: counts[nearest[i]] += 1 (counts zeroed by the caller), or with sample weights W[C] = compensated
// fp32 sums of w per candidate in a fixed order (keys_out / w_out [n], start [2C], tmp: kmp_weights_bytes(n) bytes)
cudaError_t launch_kmp_counts(const uint32_t* nearest, uint32_t n, uint32_t* counts, cudaStream_t st);
size_t kmp_weights_bytes(uint32_t n);
cudaError_t launch_kmp_weights(const uint32_t* nearest, const float* w, uint32_t n, uint32_t C, uint32_t* keys_out,
                               float* w_out, uint32_t* start, void* tmp, size_t tmp_bytes, float* W, cudaStream_t st);

// ---- mini-batch k-means (minibatch.cu) --------------------------------------------------------------------------------
// the key of one step's draws: mix(mix(tag ^ seed) + step); the tags keep the batch draw and the reassignment draw apart
// from each other and from the k-means|| draws (whose first-level inputs stay below 2^40)
constexpr uint64_t kMbTagBatch = 0x6D696E6962617463ull;      // "minibatc"
constexpr uint64_t kMbTagReassign = 0x7265617373696721ull;   // "reassig!"
constexpr uint64_t kGppTagTrial = 0x677265656479212Bull;     // "greedy!+": the trial draws of greedy k-means++
// the init stage of a mini-batch run (Job::minibatch_init): the seeding subset of init r (step = r) and the validation
// rows (step 0)
constexpr uint64_t kMbTagInit = 0x6D62696E69747375ull;       // "mbinitsu"
constexpr uint64_t kMbTagValid = 0x6D6276616C696421ull;      // "mbvalid!"
uint64_t mb_step_key(uint32_t seed, uint64_t step, uint64_t tag);

// ---- greedy k-means++ seeding (greedy_plusplus.cu) ------------------------------------------------------------------
constexpr uint32_t kGppMaxTrials = 32;
// Round state on the device: the trial whose d' column the next draw folds into d (UINT32_MAX: none), the global row
// whose d the next draw sets to 0 (UINT32_MAX: none), and stop = 1 once no row has mass left (one GPU).
struct GppCtl {
  uint32_t winner, chosen, stop, pad;
};
// the draw key of round `round`: trial t of row i draws u = ((mix(mix(key + t) ^ i) >> 11) + 0.5) 2^-53
uint64_t gpp_round_key(uint32_t seed, uint32_t round);
uint32_t gpp_draw_blocks(uint32_t n);    // bkey / brow hold L * gpp_draw_blocks(n) entries
uint32_t gpp_trial_blocks(uint32_t n);   // bsum holds L * gpp_trial_blocks(n) partials
// fold + draw: d = winner's d' column (or d), d[chosen] = 0, then keys[t] / rows[t] = the minimum (-ln u / w d^2, global
// row) of trial t over the shard (INFINITY / UINT32_MAX when no row has mass).  single: ctl_w->stop = 1 in that case.
// `ctl` and `ctl_w` are the same buffer (read-only in the draw kernel)
cudaError_t launch_gpp_draw(float* dists, const float* dprime, const float* w, uint32_t n, uint32_t off, uint32_t L,
                            const GppCtl* ctl, uint64_t rkey, double* bkey, uint32_t* brow, double* keys,
                            uint32_t* rows, GppCtl* ctl_w, bool single, cudaStream_t st);
// T[t][:] = X[rows[t] - off][:] (the trial rows live on this shard: one GPU)
cudaError_t launch_gpp_gather(const float* X, uint32_t off, int D, const uint32_t* rows, uint32_t L, const GppCtl* ctl,
                              float* T, cudaStream_t st);
// dprime[t][i] = min(d_i, true distance of row i to T[t]) (0 on trial_rows[t], d on NaN rows), bsum[t][b] = block
// partials of sum w d'^2
cudaError_t launch_gpp_trial(int metric, const float* X, uint32_t n, uint32_t off, int D, const float* T, uint32_t L,
                             const uint32_t* trial_rows, const float* dists, const float* w, const GppCtl* ctl,
                             float* dprime, double* bsum, cudaStream_t st);
// phis[t] = the partials of trial t folded in a fixed order; pick: the argmin goes to ctl, *row_log, *phi_log and its
// row to crow[D] (one GPU)
cudaError_t launch_gpp_pick(const double* bsum, uint32_t n, uint32_t L, GppCtl* ctl, const uint32_t* trial_rows,
                            double* phis, bool pick, const float* X, uint32_t off, int D, float* crow,
                            uint32_t* row_log, double* phi_log, cudaStream_t st);
// rows[j] = floor(u(key, j) * N), j < b
cudaError_t launch_mb_draw(uint32_t N, uint32_t b, uint64_t key, uint32_t* rows, cudaStream_t st);
// bsum[mb_blocks(n)] = block partials of sum w_j * (Kahan sum of (X[rows[j]] - C[a_j])^2), a_j = result[j],
// w_j = w[rows[j]] (1 without weights); keys[j] = a_j, or K when result[j] is not a centroid (such an entry has no
// inertia and no member sum)
uint32_t mb_blocks(uint32_t n);
cudaError_t launch_mb_inertia(const float* X, const uint32_t* rows, uint32_t n, int D, const float* C, uint32_t K,
                              const uint32_t* result, const float* w, uint32_t* keys, double* bsum, cudaStream_t st);
// Cnew = (C W + S) / (W + Wb) per centroid with Wb > 0 (else C), Wnew = W + Wb; Wb = wsums, or the member counts
// when wsums is nullptr (unweighted: a weight of 1 per entry)
cudaError_t launch_mb_blend(const float* C, const double* W, const float* S, const float* wsums,
                            const uint32_t* counts, uint32_t K, int D, float* Cnew, double* Wnew, cudaStream_t st);
// random reassignment of the centroids of low weight (minibatch.cu), entries drawn from X[rows[j]] with weight
// w[rows[j]]; buffers: cidx_in / cidx [K], wsorted [K], ekey_in /
// ekey [b] (double), pos_in / picked [b], npos / m [1], minkept [1], tmp of mb_reassign_bytes(b, K)
struct MbReassign {
  uint32_t K, b;
  int D;
  uint64_t key;
  double ratio;
  const float* w;          // [N] sample weights, nullptr = 1
  const float* X;          // [N][D]
  const uint32_t* rows;    // [b] the step's entries
  float* C;     // [K][D], updated in place
  double* W;    // [K], updated in place
  uint32_t *cidx_in, *cidx, *pos_in, *picked, *npos, *m;
  double *wsorted, *ekey_in, *ekey, *minkept;
  void* tmp;
  size_t tmp_bytes;
};
size_t mb_reassign_bytes(uint32_t b, uint32_t K);
cudaError_t launch_mb_reassign(const MbReassign& r, cudaStream_t st);
// out[0] = sum_c ||Cnew_c - Cold_c||^2 (double, fixed order), out[1] = #{W_c == 0}; dsq: [K] scratch
cudaError_t launch_mb_stats(const float* Cold, const float* Cnew, const double* W, uint32_t K, int D, double* dsq,
                            double* out, cudaStream_t st);
// one shard's share of the per-feature variance (Job::mean_variance): out[D] = the column sums of x_f (mean == nullptr)
// or of (x_f - mean_f)^2 over X[n][D], in double, in a fixed order; work: col_sums_doubles(D) doubles
size_t col_sums_doubles(int D);
cudaError_t launch_col_sums(const float* X, uint32_t n, int D, const double* mean, double* work, double* out,
                            cudaStream_t st);
// out[0] = sum_c ||Cnew_c - Cold_c||^2 (double, fixed order, a centroid whose term is not finite adds 0); dsq: [K]
// scratch.  The centre shift of scikit-learn's stopping rule (Job::lloyd, DESIGN.md §4p)
cudaError_t launch_center_shift(const float* Cold, const float* Cnew, uint32_t K, int D, double* dsq, double* out,
                                cudaStream_t st);

// ---- bisecting k-means (bisecting.cu) -----------------------------------------------------------------------------------
// The draws of a node [lo, hi) of perm: row i of init r in stage s draws u = unit_oo(mix(bk_node_key(seed, lo, hi, r, s)
// ^ i)), so a node's bisection is the same whenever it is computed
constexpr uint64_t kBkTagNode = 0x6269736563742121ull;   // "bisect!!"
constexpr uint32_t kBkChunk = 2048;   // positions per chunk of the fixed-order sums (and per CTA of the row kernels)
constexpr uint32_t kBkRun = 0, kBkFinal = 1;   // segment modes: E + M step; the last E step (no M step)
uint64_t bk_node_key(uint32_t seed, uint32_t lo, uint32_t hi, uint32_t r, uint32_t stage);
// one (node, init r) of a wave: positions [lo, hi) of perm, label plane r, centre slots cur / nxt of the centre buffer
// ([slot][2][D] floats, squared norms [slot][2]), chunk partials from chunk index pbase on, draw key
struct BkSeg {
  uint32_t lo, hi, r, mode, cur, nxt, pbase, seed;
  uint64_t key;
};
struct BkKey {
  double key;
  uint32_t row, pad;
};
struct BkChunkStat {
  unsigned long long fk[2];   // per child: max of (bits of e) << 32 | ~row over the rows of positive weight
  uint32_t cnt[2], npos[2], changed, pad;
};
// per segment, after a step: per child W = sum w, I = sum w e, row counts and rows of positive weight, over the labels
// of this E step; inertia = sum w e over all rows; changed labels; relocated (init_row[0] = the row); shift = sum
// ||c_new - c_old||^2.  After the init: init_row = the two centre rows (init_row[1] = UINT32_MAX: no init)
struct BkStatus {
  double W[2], I[2], inertia, shift;
  uint32_t cnt[2], npos[2], changed, relocated, init_row[2];
};
struct BkLaunch {
  const float* X;
  int D;
  uint32_t N;
  const float* w;          // nullptr = unweighted
  const uint32_t* perm;
  uint8_t* lab;            // [n_init][N] label bytes by position
  const BkSeg* segs;
  uint32_t nseg;
  const uint2* work;       // {segment, chunk} per CTA
  uint32_t nwork;
  float* cbuf;
  float* csq;
  double* part;            // [chunks][bk_partial_doubles(D)]
  BkChunkStat* cstat;      // [chunks]
  BkKey* keys;             // [chunks][2]
  BkStatus* status;        // [nseg]
  // greedy init only
  float* dist;             // [n_init][N] distance to c0 by position
  BkKey* tkeys;            // [chunks][kGppMaxTrials]
  double* phi;             // [chunks][kGppMaxTrials]
  uint32_t* trows;         // [nseg][kGppMaxTrials]
};
size_t bk_partial_doubles(int D);
cudaError_t launch_bk_iota(uint32_t* perm, uint32_t n, cudaStream_t st);
// init of every segment.  L == 0, random: centres = the two positive-weight rows of smallest -ln(u) / w.  L > 0, greedy
// k-means++ with L trials: c0 = the first of them, c1 = §4m's round 1 restricted to the node
cudaError_t launch_bk_init(const BkLaunch& a, uint32_t L, cudaStream_t st);
// one E step (and M step in mode kBkRun) of every segment: labels, new centres in slot nxt, status records
cudaError_t launch_bk_step(const BkLaunch& a, cudaStream_t st);
// applies the splits listed as segments (label plane r): perm_out = perm with each range stably partitioned by label
size_t bk_split_bytes(uint32_t N);
cudaError_t launch_bk_split(const BkLaunch& a, uint32_t* flags, uint32_t* excl, void* tmp, size_t tmp_bytes,
                            uint32_t* perm_out, cudaStream_t st);
cudaError_t launch_bk_assign(const uint32_t* perm, uint32_t N, const uint32_t* leaf_lo, uint32_t K, uint32_t* assign,
                             cudaStream_t st);

// ---- relocation of empty clusters (relocate.cu) ------------------------------------------------------------------------
// keys[i] of the shard rows i < n (global row off + i): orderable bits of d_i (L2: the Kahan sum of squared differences
// to C[assign[i]] before the square root; angular: distance_exact<1>) << 32 | ~(off + i), so that a descending order is
// (d desc, row asc); 0 when assign[i] >= K, w[i] <= 0 (w optional) or d_i is not finite
cudaError_t launch_reloc_keys(int metric, const float* X, uint32_t n, int D, const float* C, uint32_t K,
                              const uint32_t* assign, const float* w, uint32_t off, uint64_t* keys, cudaStream_t st);
// inertia of the shard (restarts, DESIGN.md §4n): *out = sum of w_i e_i over the rows a key of launch_reloc_keys would
// call eligible, e = that key's d (L2) or d^2 (angular), in double; bsum holds inertia_blocks(n) block partials, folded
// by launch_fixed_sum
uint32_t inertia_blocks(uint32_t n);
cudaError_t launch_inertia(int metric, const float* X, uint32_t n, int D, const float* C, uint32_t K,
                           const uint32_t* assign, const float* w, double* bsum, double* out, cudaStream_t st);
struct RelocState {
  uint64_t prefix, thr;   // digits fixed so far; the selection threshold
  uint32_t above, done, eligible, pad;
};
// top[0 .. T) = the T largest non-zero keys of keys[n], descending, 0 after the last one; state->eligible = the number
// of non-zero keys.  Buffers: state [1], hist [256], sel / top [cap = reloc_cap(T)], nsel [1], tmp of
// reloc_select_bytes(n, cap) bytes
struct RelocSelect {
  uint32_t n, T, cap;
  const uint64_t* keys;
  RelocState* state;
  uint32_t* hist;
  uint64_t *sel, *top;
  uint32_t* nsel;
  void* tmp;
  size_t tmp_bytes;
};
uint32_t reloc_cap(uint32_t T);
size_t reloc_select_bytes(uint32_t n, uint32_t cap);
cudaError_t launch_reloc_select(const RelocSelect& s, cudaStream_t st);
// meta[2j] = assign of the row of top[j] (local row ~low word - off), meta[2j + 1] = its weight's bits (1 without w)
cudaError_t launch_reloc_gather(const uint64_t* top, uint32_t T, uint32_t off, const uint32_t* assign, const float* w,
                                uint32_t* meta, cudaStream_t st);
// the r relocations in walk order, meta[3j] = empty cluster, [3j + 1] = donor, [3j + 2] = weight bits, xs [r][D] the
// rows: sums[donor] -= w x, counts[donor] -= 1, wsums[donor] -= w (wsums optional); sums[e] = w x, counts[e] = 1,
// wsums[e] = w
cudaError_t launch_reloc_apply(float* sums, uint32_t* counts, float* wsums, int D, const float* xs,
                               const uint32_t* meta, uint32_t r, cudaStream_t st);
// angular, after the normalisation: C[e] = x / ||x|| in the reference's order
cudaError_t launch_reloc_cos_overwrite(float* C, int D, const float* xs, const uint32_t* meta, uint32_t r,
                                       cudaStream_t st);

cudaError_t launch_half_to_float(const void* src, float* dst, size_t n, cudaStream_t st);
cudaError_t launch_float_to_half(const float* src, void* dst, size_t n, cudaStream_t st);
cudaError_t launch_fill_u32(uint32_t* p, uint32_t v, size_t n, cudaStream_t st);
// *out = bsum[0] + ... + bsum[nb - 1], added in an order that depends only on nb (fixed_order.cuh)
cudaError_t launch_fixed_sum(const double* bsum, uint32_t nb, double* out, cudaStream_t st);

// ---- k-NN ------------------------------------------------------------------------------------------
// inverse assignments: inv[] = sample ids sorted by (cluster, id), off[K+1] = CSR offsets
cudaError_t launch_knn_inverse(const uint32_t* assign, uint32_t n, uint32_t K, uint32_t* iota,
                               uint32_t* keys_out, uint32_t* inv, uint32_t* off, uint32_t* counts,
                               UpdateWorkspace& ws, cudaStream_t st);
cudaError_t launch_knn_radii(int metric, const float* X, const float* C, uint32_t n, int D, uint32_t K,
                             const uint32_t* assign, float* radii, cudaStream_t st);
cudaError_t launch_knn_centroid_distances(int metric, const float* C, uint32_t K, int D, float* cd,
                                          cudaStream_t st);
cudaError_t launch_knn_search(int metric, int k, const float* X, const float* C, uint32_t N, int D,
                              uint32_t K, uint32_t q_offset, uint32_t q_length, const uint32_t* assign,
                              const uint32_t* inv, const uint32_t* inv_off, const float* cd,
                              const float* radii, float* heap_scratch, uint32_t* neighbors,
                              unsigned long long* d_pairs, const uint32_t* rows, const uint32_t* d_nrows,
                              cudaStream_t st);
cudaError_t launch_knn_radii_fix(const uint32_t* inv_off, uint32_t K, float* radii, cudaStream_t st);
cudaError_t launch_knn_tail_rows(const uint32_t* inv, uint32_t nv, uint32_t n, uint32_t* rows, uint32_t* d_nrows,
                                 cudaStream_t st);

// ---- tensor-core filter (assign_tc.cu) -----------------------------------------------------------
struct TcPlan;  // opaque; owns the fp16 centroid table, tensor maps, queues
bool tc_supported(int metric, uint32_t n, int D, uint32_t K);
// multiprocessors of the current device: the grid size unit of the grid-stride kernels
unsigned device_sms();
cudaError_t tc_plan_create(TcPlan** plan, int metric, uint32_t max_n, int D, uint32_t K, int device);
void tc_plan_destroy(TcPlan* plan);
// one full assignment pass.  assign == nullptr: result[i] as launch_assign_exact would produce it.  Otherwise the
// pass's bookkeeping (launch_finalize_assign) is fused: prev[i] = assign[i], assign[i] = winner, *d_changed +=
// changes; result[] is then scratch for the few rows that take the exact full pass.
// compute_csq: csq[] (the caller's buffer, K floats) is filled by the pass's own preparation launch (what launch_csqr
// would write) instead of being read as an input.
cudaError_t tc_assign(TcPlan* plan, const float* X, const float* C, const float* csq, uint32_t n,
                      uint32_t* result, uint32_t* assign, uint32_t* prev, uint32_t* d_changed, cudaStream_t st,
                      bool compute_csq = false);
// mini-batch pass over a row list (tc_assign_kernel<NKB, 0, true>): result[i] = the winner of sample rows[i], i < n, as
// launch_assign_exact defines it; X has nX rows; row_result [nX] is scratch of the exact list pass (indexed by row)
cudaError_t tc_assign_rows(TcPlan* plan, const float* X, uint32_t nX, const uint32_t* rows, uint32_t n, const float* C,
                           const float* csq, uint32_t* result, uint32_t* row_result, cudaStream_t st);
// statistics of the last pass (for logging / bench): queue length and overflow rows
void tc_last_stats(TcPlan* plan, uint32_t* n_recheck, uint32_t* n_overflow);
// Yinyang local step (assign_tc.cu): candidate pairs with exact true distances for the listed rows
struct TcQueues {
  const uint32_t* rowq;       // [3*i]: row, first pair, pair count
  const uint32_t* d_nrowq;
  const uint32_t* pair_cand;
  const float* pair_score;    // exact distance of (row, pair_cand)
  const uint32_t* ovf_rows;   // rows the filter could not bound
  const uint32_t* d_novf;
};
// every plan also serves the Yinyang local step and bounds refresh (MODE 1 / 3), at every D it supports
// (512 < D <= 1024 on 64-row tiles)
cudaError_t tc_yy_candidates(TcPlan* plan, const float* X, const float* C, const float* csq, uint32_t n,
                             const uint32_t* rows, const uint32_t* d_nrows, cudaStream_t st);
cudaError_t tc_exact_distances(TcPlan* plan, const float* X, const float* C, uint32_t n, const uint32_t* pair_row,
                               const uint32_t* pair_cand, const uint32_t* d_npairs, uint32_t max_pairs,
                               float* pair_score, cudaStream_t st);
void tc_queues(TcPlan* plan, TcQueues* q);
// Yinyang bounds refresh on the tensor cores (assign_tc.cu, MODE 3): tc_yy_layout once per grouping (host map
// centroid -> group), then tc_yy_refresh per refresh; rows left on the overflow list need launch_yy_init_rows
cudaError_t tc_yy_layout(TcPlan* plan, const uint32_t* host_groups, uint32_t G);
// the host part of tc_yy_layout (pure function): table row -> centroid (UINT32_MAX = padding), group of every
// 4-row quad, CSR of the group members, number of 128-row n-tiles
void tc_yy_layout_host(const uint32_t* host_groups, uint32_t K, uint32_t G, std::vector<uint32_t>* perm,
                       std::vector<uint32_t>* qgroup, std::vector<uint32_t>* goff, std::vector<uint32_t>* gmem,
                       int* nt3);
bool tc_yy_layout_ready(TcPlan* plan, uint32_t G);
cudaError_t tc_yy_refresh(TcPlan* plan, const float* X, const float* C, const float* csq, uint32_t n,
                          const uint32_t* assign, const uint32_t* groups, uint32_t G, float* bounds, cudaStream_t st);
// k-NN candidate search on the tensor cores (assign_tc.cu); see the comment there
bool tc_knn_supported(int metric, int k, uint32_t N, int D, uint32_t K);
// metric 1 (angular): candidates come from the L2 pass (cd / radii must then be the L2 quantities), the margin is
// widened by the samples' deviation from unit length, exact distances and the selection use the angular metric; if the
// samples are not unit vectors (deviation > 1e-2) *h_error is set and the caller has to run the exact search
cudaError_t tc_knn_search(int metric, int k, const float* X, const float* C, uint32_t N, int D, uint32_t K,
                          const uint32_t* assign, const uint32_t* inv, const uint32_t* off, const float* cd,
                          const float* radii, uint32_t nv, uint32_t* neighbors, uint32_t* fb_rows, uint32_t* d_nfb,
                          unsigned long long* d_pairs, uint32_t* h_error, uint32_t part, uint32_t nparts,
                          cudaStream_t st);
// several GPUs: every device serves part `part` of `nparts` of the query tiles into its own full-size neighbour
// array (pre-filled with 0xFFFFFFFF); the arrays are merged with an element-wise minimum over peer memory
struct PeerU32 {
  int n;
  const uint32_t* p[kMaxPeers];
};
cudaError_t launch_peer_min_u32(const PeerU32& pb, size_t count, uint32_t* out, cudaStream_t st);
// 0 = clean; 0x1000+site = a pipeline wait timed out at `site` (results of that pass are invalid)
uint32_t tc_last_error(TcPlan* plan);
uint32_t tc_last_pairs(TcPlan* plan);
void tc_set_capture(TcPlan* plan, bool on);   // the next tc_assign is recorded into a CUDA graph (stream capture)
int tc_kernel_times(TcPlan* plan, float* ms_out, int max_out);

}  // namespace kmb
