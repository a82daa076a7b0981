// assign_tc.cu -- the H100 hot path: samples x centroids L2 ranking as a dense fp16 contraction on
// the Hopper tensor cores (wgmma), fused with a per-sample candidate filter; the exact fp32 re-check
// (below + simt_kernels.cu) then makes the final, reference-identical decision.
//
// What the reference does here: kmeans_assign_lloyd (reference src/kmeans.cu:293-364) -- one CUDA
// thread per sample, N*K*D Kahan-compensated round-down FMAs on the FP32 pipe.
//
// What this file does instead, per persistent CTA (one per SM) and per tile of 128 samples:
//   converter warps : one thread per sample row: fp32 row from global memory -> *s (power of two) -> fp16 ->
//                     the A operand in shared memory (128-byte swizzled K-major, the layout wgmma reads); per
//                     row ||x~||, ||x - x~|| are accumulated for the error bound
//   B producer      : TMA streams the fp16 centroid table (128 centroids x 64 features per stage,
//                     128B swizzle) + the per-n-tile bias block through mbarrier rings
//   consumer warps  : two warpgroups, one per 64-row half of the tile; each issues wgmma m64n128k16 (A and B
//                     from shared memory, fp32 accumulators in its registers) over every K-block, plus one
//                     extra K=16 step that adds -||c||^2/2 as three fp16 terms against constant ones, so
//                     acc = x.c - ||c||^2/2.  The epilogue works on the accumulator fragment as it lands: a
//                     lane holds 32 columns of each of two rows, and the four lanes of a quad hold all 128
//                     columns of their rows.  The running row maximum M is updated (quad all-reduce of the
//                     lanes' chunk maxima) and every column whose value is within `margin` of M is recorded (a
//                     32-bit mask per row and lane, decoded into columns by the emitters); margin is a rigorous bound on
//                     |approx - exact| derived from the actual rounding residuals (Cauchy-Schwarz), so the
//                     reference's fp32 winner is guaranteed to be among the recorded candidates.
//   rows with one candidate are final; rows with several go to the exact re-check queue; rows with
//   non-finite data or too many candidates go to the exact full pass.  Assignments are therefore
//   bit-identical to the reference kernel's, ties included.
//
// Shared memory (227 KB per block on H100) holds the whole fp16 A operand of a tile (16 KB per 64 features), so
// 128-row tiles serve D <= 512.  The A region is a ring of K-block slots with room for more than one tile
// (D <= 256), so the next tile's first K-blocks are converted while the current one is multiplied.  For D > 256 the
// pipeline is shallower (see smem_layout).  512 < D <= 1024 (every MODE) uses tiles of 64 rows (8 KB per 64
// features); both consumer warpgroups then hold the same rows, each one 64-column half of every n-tile (tile64 below).
//
// The same kernel template serves two more callers (MODE template parameter, see tc::Params):
//   MODE 1  Yinyang local step (reference kmeans.cu:584-672): the samples are a compacted row list; candidates =
//           every centroid within the margin of the row's SECOND best; all of them get their exact true distance
//           (yinyang.cu finishes the step).
//   MODE 2  k-NN (reference knn.cu:177-347): queries and candidates are the samples in a cluster-aligned table;
//           a tile is multiplied with one segment per candidate cluster, both operands centred on that
//           cluster's centroid; the epilogue keeps the k+1 largest 4-column-group maxima per half-row as its
//           threshold and records candidate masks in global lists (namespace knn below has the passes around it).
//           64-row tiles: a row has four parts of 32 columns (two per warpgroup) instead of two halves.
#include <cuda.h>
#include <cuda_fp16.h>

#include <cstdio>
#include <algorithm>
#include <array>
#include <cstring>
#include <map>
#include <mutex>
#include <tuple>
#include <utility>
#include <vector>

#include <cub/cub.cuh>

#include "exact.cuh"
#include "kernels.h"
#include "sm90_ptx.cuh"

namespace kmb {

namespace tc {
constexpr int TM = 128;                 // samples per tile (two wgmma M = 64 halves, one per consumer warpgroup)
constexpr int TN = 128;                 // centroids per n-tile (wgmma N)
constexpr int KB = 64;                  // fp16 elements per K-block = one 128-byte swizzle row
constexpr int MAX_NKB = 8;              // D <= 512: the A operand of a tile lives in shared memory, 16 KiB per K-block
// 512 < D <= 1024 (every MODE): tiles of 64 rows, both consumer warpgroups on the same rows, each on one 64-column
// half of every n-tile (wgmma m64n64k16); an A K-block is 8 KiB, so the whole tile still stays resident
constexpr int MAX_TILE64_NKB = 16;
constexpr int MAX_A_SLOTS = 16;
constexpr int WIDE_NKB = 4;             // D > 256 ("wide"): a 128 KiB A tile leaves room for a 2-stage B ring only
constexpr int B_STAGES = 4;             // fp16 centroid stages of ONE K-block (64 features x 128 rows = 16 KiB): a stage is
                                        // refilled as soon as both warpgroups' wgmmas on it have retired
constexpr int B_KB_BYTES = TN * 128;    // one K-block of the centroid tile: 16 KiB
constexpr int B_STAGE_BYTES = B_KB_BYTES;
constexpr int AUG_B_BYTES = TN * 32;    // 4 KiB
constexpr int LIST_LEN = 5;             // entries per epilogue thread: one per n-tile in which one of its two rows held a
                                        // candidate (2 x row maximum, 2 x 32-bit mask, 16-bit n-tile)
constexpr int LIST_ARRAYS = 4;
// Knock-out builds (timing experiments only, results are garbage): 1 = the epilogue does not read the accumulators,
// 2 = no MMA is issued, 3 = converters do no work, 5 = the B / bias copies are not issued, 7 = the epilogue loads the
// accumulators but skips the ALU work on them.  Which of them shortens the kernel says what bounds it.
#ifndef KMB_KO
#define KMB_KO 0
#endif
// Four warpgroups: 0 = emitters + B producer, 1 = converters, 2 and 3 = consumers.
constexpr int FIRST_EMIT_WARP = 0;      // 3 emitter warps (merge + global emission)
constexpr int WARP_B_PRODUCER = 3;      // TMA producer: the last warp of warpgroup 0
constexpr int FIRST_CONV_WARP = 4;      // 4 converter warps
constexpr int FIRST_EPI_WARP = 8;       // 8 consumer warps = 2 warpgroups (wgmma + epilogue)
constexpr int N_CONV_WARPS = 4;
constexpr int N_EPI_WARPS = 8;
constexpr int N_EMIT_WARPS = 3;
constexpr int N_THREADS = 16 * 32;      // 512
// Registers per thread after setmaxnreg.  512 threads start at 128 (544 threads were held to 96, and every consumer
// spilled); warpgroups 0 and 1 hand registers back and the consumers, which hold 64 accumulator registers plus the
// epilogue, take them.  Each of the four register-file sub-partitions holds one warp of every warpgroup, so the four
// counts share its 512 registers per lane.
constexpr int REGS_WG0 = 64, REGS_CONV = 80, REGS_EPI = 184;
static_assert(REGS_WG0 % 8 == 0 && REGS_CONV % 8 == 0 && REGS_EPI % 8 == 0, "setmaxnreg counts are multiples of 8");
static_assert(REGS_WG0 >= 24 && REGS_CONV >= 24 && REGS_EPI >= 24 && REGS_WG0 <= 256 && REGS_CONV <= 256 &&
              REGS_EPI <= 256, "setmaxnreg counts lie in [24, 256]");
static_assert(REGS_WG0 + REGS_CONV + 2 * REGS_EPI <= 512, "one warp of each warpgroup per 16K-register sub-partition");
constexpr int MAX_CAND = 32;            // candidates per row before falling back to the full exact pass (one per lane of the finishing warp)
constexpr int KNN_CAP = 40;             // k-NN: (chunk, mask) entries per row part (half; NKB 9..16: quarter) in global memory
constexpr int KNN_MAX_KK = 16;          // k + 1 <= 16 on the tensor-core path
constexpr float SENTINEL_GUARD = -65000.f;   // padded / dead centroids score exactly -65504: thresholds below this are not trusted

// counters[] slots
enum { CNT_PAIRS = 0, CNT_ROWQ = 1, CNT_OVF = 2, CNT_ERR = 3, CNT_N = 4 };

struct Stats {       // written by the centroid prep kernels, read by the main kernel
  float scale;       // s = 2^k applied to samples and centroids before fp16 rounding
  float cmax;        // max_c ||s*c||  (finite centroids)
  float dcmax;       // max_c ||s*c - fp16(s*c)||
  uint32_t csq_max_bits;
  uint32_t force_exact; // cosine only: a centroid with an infinite element / norm can still win -> no filtering
  float yabs;           // k-NN: max over samples of s * (|y| + |c(y)|): bounds the rounding of the centring y - c
  float mun;            // s * ||mu|| (upper bound): mu = centring vector of the assignment filter (0: cosine, k-NN)
  float knn_extra;      // k-NN, angular metric served through the L2 pass: s^2 * max |1 - ||y||^2| (see tc_knn_search)
};

constexpr uint32_t LIST_ARRAY = 2 * LIST_LEN * 256 * 4;   // bytes of one of the four 32-bit list arrays (both tile parities)
constexpr uint32_t LIST_NT_BYTES = 2 * LIST_LEN * 256 * 2; // the n-tile array (16 bit: nt <= 16383, see tc_supported)
// per-tile state in the fin region, in words from the parity's base: M, margin, M2 per row; per epilogue thread its list
// length (bits 0-7) and flags (R0 in bits 8-15, R1 in bits 16-23)
enum { FIN_M = 0, FIN_MARGIN = TM, FIN_M2 = 2 * TM, FIN_STATE = 3 * TM, FIN_WORDS = 3 * TM + 256 };
struct SmemLayout {  // byte offsets from the 1024-aligned dynamic smem base
  uint32_t a, b, aug_a, aug_b, list, norms, fin, mu, bars, total;
};

// Per-shape pipeline depths.  The A region is a ring of a_slots(nkb) K-block slots that the converters fill K-block by
// K-block, across tile boundaries: with more slots than K-blocks per tile, the next tile's first K-blocks are converted
// while the current tile is still being multiplied.  D <= 128: 4 slots (two tiles or more), 4 B stages, 2 bias buffers.
// D 129-256: 5-6 slots, 4 B stages, 1 bias buffer.  D > 256: the 128 KiB region (8 slots) leaves 2 B stages and 1 bias
// buffer.  The norms ring must be deeper than the number of segments the converters can run ahead (see layouts_fit).
__host__ __device__ constexpr bool wide_nkb(int nkb) { return nkb > WIDE_NKB; }
__host__ __device__ constexpr int b_stages(int nkb) { return wide_nkb(nkb) ? 2 : B_STAGES; }
__host__ __device__ constexpr int aug_bufs(int nkb) { return nkb <= 2 ? 2 : 1; }
// NKB 9..16: 16 slots of 64 rows (128 KiB), so NKB < 16 still converts the next tile's first K-blocks during this one
__host__ __device__ constexpr int a_slots(int nkb) { return nkb <= 2 ? 4 : nkb == 3 ? 5 : nkb == 4 ? 6 : nkb <= MAX_NKB ? MAX_NKB : 2 * MAX_NKB; }
__host__ __device__ constexpr bool tile64(int nkb) { return nkb > MAX_NKB; }
__host__ __device__ constexpr int tile_rows(int nkb) { return tile64(nkb) ? 64 : TM; }
__host__ __device__ constexpr int a_kb_bytes(int nkb) { return tile_rows(nkb) * 128; }   // one A K-block: 16 / 8 KiB
__host__ __device__ constexpr int mu_features(int nkb) { return (nkb > MAX_NKB ? nkb : MAX_NKB) * KB; }
// The converters write the norms of segment f + depth after waiting for the slot of its last K-block, i.e. after every
// consumer warp released K-block (f + depth + 1) * nkb - 1 - a_slots; that K-block belongs to segment f + 1 or later
// (so each warp has read the norms of f) exactly when depth * nkb > a_slots.
__host__ __device__ constexpr int norm_depth(int nkb) { return a_slots(nkb) / nkb + 1; }

__host__ __device__ constexpr SmemLayout smem_layout(int nkb) {
  SmemLayout L{};
  uint32_t o = 0;
  L.a = o; o += a_slots(nkb) * a_kb_bytes(nkb);
  L.b = o; o += b_stages(nkb) * B_STAGE_BYTES;
  L.aug_a = o; o += tile_rows(nkb) * 32;   // constant A-side bias operand: K = 16 fp16 per row, no swizzle (4 / 2 KiB)
  L.aug_b = o; o += aug_bufs(nkb) * AUG_B_BYTES;
  // candidate lists (MODE 0 / 1): 4 arrays (maximum of row R0 | of row R1 | mask of R0 | mask of R1) of
  // [tile parity][entry][epilogue thread] words, LIST_ARRAY bytes apart, then the n-tiles as 16-bit [parity][entry][thread].
  // MODE 2 reuses [list, norms) as its top-kk / bucket scratch: 48 rows x 256 x 4 bytes (static_assert below)
  L.list = o; o += LIST_ARRAYS * LIST_ARRAY + LIST_NT_BYTES;
  L.fin = o; o += 2 * FIN_WORDS * 4;  // [tile parity][FIN_*]
  L.norms = o; o += norm_depth(nkb) * 4 * TM * 4;   // [segment % depth][x|d][row]  x~^2 | residual^2 | (k-NN) exact s^2|x-c|^2 | (k-NN) s^2(|x|+|c|)^2
  L.mu = o; o += mu_features(nkb) * 4;   // -mu * s per feature (zero padded): the converters' centring term
  L.bars = o; o += 64 * 8;
  L.total = o;
  return L;
}
static_assert(LIST_ARRAYS * LIST_ARRAY + LIST_NT_BYTES + 2 * FIN_WORDS * 4 >= 48 * 256 * 4, "k-NN scratch overlaps the norms");
__host__ __device__ constexpr bool layouts_fit() {
  for (int k = 1; k <= MAX_TILE64_NKB; k++)
    if (smem_layout(k).total + 1024 > 232448 || a_slots(k) < k || a_slots(k) > MAX_A_SLOTS || norm_depth(k) * k <= a_slots(k))
      return false;
  return true;
}
static_assert(layouts_fit(), "227 KiB of shared memory per block on H100; a whole tile in the A ring; norms ring depth");
// the 64-row layout (A 128 KiB, B 32 KiB, bias 2 + 4 KiB, lists and per-tile state 50 KiB, norms 4 KiB, -mu s NKB / 4
// KiB, barriers, alignment): 226816 + 256 NKB bytes of the 232448 an H100 block may opt in to
__host__ __device__ constexpr bool tile64_budget() {
  for (int k = MAX_NKB + 1; k <= MAX_TILE64_NKB; k++)
    if (smem_layout(k).total + 1024 != 226816u + 256u * k) return false;
  return true;
}
static_assert(tile64_budget(), "64-row tile budget");

// barrier indices inside the bars[] array
enum {
  BAR_B_FULL = 0,                             // [B_STAGES]
  BAR_B_EMPTY = BAR_B_FULL + B_STAGES,        // [B_STAGES]
  BAR_AUG_FULL = BAR_B_EMPTY + B_STAGES,      // [2]
  BAR_AUG_EMPTY = BAR_AUG_FULL + 2,           // [2]
  BAR_A_FULL = BAR_AUG_EMPTY + 2,             // [a_slots] converters -> consumers, per A slot
  BAR_A_FREE = BAR_A_FULL + MAX_A_SLOTS,      // [a_slots] consumers -> converters, per A slot
  BAR_EMIT_FULL = BAR_A_FREE + MAX_A_SLOTS,   // [2] epilogue -> emitter (per tile parity)
  BAR_EMIT_EMPTY = BAR_EMIT_FULL + 2,         // [2]
  BAR_COUNT = BAR_EMIT_EMPTY + 2
};
static_assert(BAR_COUNT <= 63, "barrier array too small");   // slot 63 is the CTA's "a wait has given up" flag

// Every field defaults to 0 / nullptr (one device: knn_nparts = 1); a pass sets the fields its MODE reads.
struct Params {
  uint32_t n = 0;
  int D = 0;
  uint32_t K = 0;
  int nkb = 0;                   // K-blocks of 64 features
  int nt = 0;                    // n-tiles of 128 centroids
  uint32_t ntiles = 0;           // sample tiles
  const __half* aug_blob = nullptr;   // [nt][AUG_B_BYTES] in the shared-memory byte layout
  const Stats* stats = nullptr;
  uint32_t* result = nullptr;    // [n]
  uint32_t* pair_row = nullptr;  // re-check queue: (row, candidate) pairs
  uint32_t* pair_cand = nullptr;
  uint32_t max_pairs = 0;
  uint32_t* rowq = nullptr;      // [3*i]: row, first pair, pair count
  uint32_t* ovf_rows = nullptr;  // rows for the full exact pass
  uint32_t* counters = nullptr;  // CNT_*
  int metric = 0;                // 0 = L2 (score x.c - ||c||^2/2), 1 = cosine (score x.c; larger dot = smaller angle)
  const float* neg_mu_s = nullptr;   // [nkb*64] -mu*s (zero padded), nullptr = no centring: MODE 0/1 multiply
                                     // (x - mu) with the table of (c - mu); scores shift by a per-row constant, so the
                                     // ranking is unchanged while the fp16 rounding error (proportional to
                                     // |x - mu| |c - mu|) shrinks
  // MODE 0 with assign != nullptr: the bookkeeping of the assignment pass is fused (reference kmeans.cu:356-363):
  // prev[row] = assign[row]; assign[row] = winner; *d_changed += (winner != old); rows that go to the re-check /
  // exact queues are finished by those kernels
  uint32_t* assign = nullptr;
  uint32_t* prev = nullptr;
  uint32_t* d_changed = nullptr;
  // MODE 3 (Yinyang bounds refresh, reference kmeans_yy_init kmeans.cu:431-485): the table is the GROUP-SORTED
  // centroid list, every group padded to whole 4-column quads (yy_qgroup[(n-tile * 2 + half) * 16 + quad] = group of
  // that quad, UINT32_MAX past the end).  The epilogue folds the quad maxima into per-group maxima and turns each
  // into a LOWER bound of the distance to the nearest centroid of that group, d >= sqrt(|x^|^2 - 2 (max + E)) / s,
  // merged into bounds[row][1 + g] with an atomic minimum; the sample's own group and its upper bound are exact
  // (yy_own_group_kernel).  Valid bounds are all Yinyang needs: the assignments stay those of Lloyd's algorithm.
  const uint32_t* yy_qgroup = nullptr;
  const uint32_t* yy_groups = nullptr;   // [K] centroid -> group
  const uint32_t* yy_assign = nullptr;   // [n]
  float* yy_bounds = nullptr;            // [n][G + 1]
  uint32_t G = 0;
  // MODE 1 (Yinyang local step): the samples are the rows listed in rows[0 .. *d_nrows), read straight from
  // global memory by the converter warps; every column within the margin of the row's SECOND best score is a
  // candidate and every candidate goes to the pair queue (the caller needs exact best and second-best distances)
  const float* X = nullptr;
  const uint32_t* rows = nullptr;
  const uint32_t* d_nrows = nullptr;
  // MODE 2 (k-NN candidate pass): queries AND candidates are the samples in the cluster-aligned table order: cluster
  // c owns the blocks [blk_first[c], blk_first[c+1]) of 128 table rows (zero-padded), rows[] maps a table row to the
  // original sample (UINT32_MAX = padding), so query tile t IS block t.  A tile is multiplied with a list of
  // SEGMENTS knn_ranges[knn_roff[t] .. +knn_rcount[t]): each segment is the block range of ONE candidate cluster B,
  // and for it the queries are re-converted relative to B's centroid -- both operands are then small vectors
  // (x - c_B, y - c_B), which is what gives the fp16 product enough resolution inside tight clusters.  The per-row
  // constant s^2 |x - c_B|^2 / 2 is folded into the threshold, so everything the epilogue keeps (top-kk list, entry
  // maxima) lives in the translation-invariant score g = -s^2 d^2 / 2.  Every column within the margin of the row's
  // kk-th largest 4-column-group maximum (kk = k + 1, self included) is recorded as (max, mask, chunk id, margin).
  // 64-row tiles (NKB 9..16): query tile t is half t & 1 of block t >> 1; the per-tile arrays below stay per block and
  // are read at t >> 1, so the kernel runs 2 * (blocks) tiles and skips a second half without live rows.
  const uint32_t* d_ntiles = nullptr;
  const uint32_t* tile_nrows = nullptr;
  const uint32_t* blk_cluster = nullptr;
  const float* C = nullptr;                // centroids [K][D] (fp32)
  const uint2* knn_ranges = nullptr;
  const uint32_t* knn_roff = nullptr;
  const uint32_t* knn_rcount = nullptr;
  const uint32_t* knn_nblk = nullptr;      // blocks per tile (sum over its segments)
  int kk = 0;
  int knn_first_pass = 0;        // 1: the per-row state starts empty; the tile has TWO segments, both its own cluster:
                                 //    the first sweep only builds the top-kk threshold, the second one only records
  uint32_t knn_stride = 0;       // = parts * (table rows): stride of the [kk][stride] top-kk state (2 parts per row,
                                 //   4 at NKB 9..16)
  float* knn_topk = nullptr;     // [kk][stride] descending group maxima (g-space) of part (table row * parts + part)
  uint32_t* knn_cnt = nullptr;   // [stride] entries used
  uint32_t* knn_flags = nullptr; // [stride]
  float* knn_dub = nullptr;      // [stride] upper bound of the exact distance to the kk-th nearest candidate so far
  uint4* knn_entries = nullptr;  // [stride][KNN_CAP]: (group max bits (g-space), mask, chunk id, margin bits)
  uint32_t knn_part = 0, knn_nparts = 1;   // query-tile shard of this device (0, 1 = everything)
};

// ---------------------------------------------------------------------------------------------------
// centroid preparation: scale, fp16 table (zero padded to [nt*256][nkb*64]), bias blobs, statistics
// ---------------------------------------------------------------------------------------------------
__global__ void tc_prep_stats_kernel(const float* __restrict__ csq, uint32_t K, Stats* __restrict__ st) {
  // max finite ||c||^2 (positive floats order like unsigned ints)
  uint32_t best = 0;
  for (uint32_t c = blockIdx.x * blockDim.x + threadIdx.x; c < K; c += gridDim.x * blockDim.x) {
    float v = csq[c];
    if (v == v && v < 3.0e38f) best = max(best, __float_as_uint(fmaxf(v, 0.f)));
  }
  for (int o = 16; o > 0; o >>= 1) best = max(best, __shfl_xor_sync(0xffffffffu, best, o));
  if ((threadIdx.x & 31) == 0) atomicMax(&st->csq_max_bits, best);
}

// s = 2^k with s * cmax in [32, 64); 1 when cmax is 0 or not finite
__device__ __forceinline__ float prep_scale(float cmax) {
  float s = 1.f;
  if (cmax > 0.f && cmax < 3.0e38f) {
    int e;
    frexpf(cmax, &e);          // cmax = m * 2^e, m in [0.5, 1)
    s = ldexpf(1.f, 6 - e);    // s*cmax in [32, 64)
  }
  return s;
}

// k-NN (one thread): scale and norm bound of the table from tc_prep_stats_kernel's maximum; the caller zeroes the
// Stats, and the table kernel raises dcmax from there
__global__ void tc_prep_scale_kernel(Stats* __restrict__ st) {
  const float cmax = __fsqrt_ru(__uint_as_float(st->csq_max_bits));
  const float s = prep_scale(cmax);
  st->scale = s;
  st->cmax = cmax * s * 1.001f;
}

// bias of table row `row`: h as three fp16 terms, or -65504 for a padding / invalid row, in the row's slot of the
// K = 16 no-swizzle block (core matrix = 8 rows x 16 bytes contiguous, 8-row groups 128 bytes apart, second K half
// TN*16 bytes further)
__device__ __forceinline__ void write_bias_row(__half* __restrict__ aug_blob, uint32_t row, bool valid, float h) {
  __half b[3];
  if (valid) {
    b[0] = __float2half_rn(h);
    const float r1 = h - __half2float(b[0]);
    b[1] = __float2half_rn(r1);
    b[2] = __float2half_rn(r1 - __half2float(b[1]));
  } else {
    b[0] = __float2half_rn(-65504.f);
    b[1] = b[2] = __float2half_rn(0.f);
  }
  const uint32_t t = row / TN, r = row % TN;
  __half* blob = aug_blob + static_cast<size_t>(t) * (AUG_B_BYTES / 2);
  for (int k = 0; k < 16; k++) {
    const int j = k >> 3, e = k & 7;
    blob[(j * (TN * 16) + (r >> 3) * 128 + (r & 7) * 16) / 2 + e] = k < 3 ? b[k] : __float2half_rn(0.f);
  }
}

// one table row (a centroid, or a zero padding row up to nt*TN) by one warp; s = Stats::scale; csq / mu may have been
// written earlier in the SAME launch by other CTAs (fused preparation), hence no __restrict__ / read-only loads on them
__device__ __forceinline__ void prep_table_row(uint32_t row, int lane, float s, int metric, const float* __restrict__ C,
                                               const float* csq, uint32_t K, int D, int nkb, __half* __restrict__ table,
                                               __half* __restrict__ aug_blob, Stats* st,
                                               const uint32_t* __restrict__ gather, const float* mu, int by_source) {
  // by_source (Yinyang refresh layout): table row r holds centroid gather[r] (UINT32_MAX = padding) and csq[] is
  // indexed by the centroid; otherwise csq[] is indexed by the table row and rows >= K are padding
  const int Dp = nkb * KB;
  uint32_t src = row;
  bool finite = row < K;
  if (by_source) {
    src = gather[row];
    finite = src != UINT32_MAX;
    if (!finite) src = 0;
  } else if (finite && gather) {
    src = gather[row];
  }
  const uint32_t qrow = by_source ? src : row;
  const float* Crow = C + static_cast<size_t>(src) * D;
  if (finite) {
    float q = __ldcg(csq + qrow);
    finite = (q == q) && q < 3.0e38f;
    for (int f = lane; f < D; f += 32) {
      float v = Crow[f];
      if (!(fabsf(v) < 3.0e38f)) finite = false;
    }
    finite = __all_sync(0xffffffffu, finite);
    if (metric == 1 && !finite) {
      // a NaN centroid never wins (acos(NaN) fails every '<'), but one with +-Inf elements or an
      // overflowing norm can: the filter has no bound for it, so the whole pass runs exact
      bool has_nan = false;
      for (int f = lane; f < D; f += 32) {
        float v = Crow[f];
        has_nan |= (v != v);
      }
      has_nan = __any_sync(0xffffffffu, has_nan);
      if (!has_nan && lane == 0) st->force_exact = 1u;
    }
  }
  float d2 = 0.f;
  for (int f = lane; f < Dp; f += 32) {
    float v = (finite && f < D) ? (mu ? Crow[f] - mu[f] : Crow[f]) * s : 0.f;
    __half h = __float2half_rn(v);
    float r = v - __half2float(h);
    d2 = fmaf(r, r, d2);
    table[static_cast<size_t>(row) * Dp + f] = h;
  }
  for (int o = 16; o > 0; o >>= 1) d2 += __shfl_xor_sync(0xffffffffu, d2, o);
  if (lane == 0) {
    if (finite) atomicMax(reinterpret_cast<uint32_t*>(&st->dcmax), __float_as_uint(__fsqrt_ru(d2) * 1.0001f));
    // bias: -(s^2 ||c - mu||^2 / 2) (L2; s = 2^k: exact; this order cannot overflow for tiny data), 0 (cosine)
    write_bias_row(aug_blob, row, finite, (finite && metric != 1) ? -0.5f * ((s * __ldcg(csq + qrow)) * s) : 0.f);
  }
}

// ---------------------------------------------------------------------------------------------------
// The whole centroid preparation of one pass as ONE launch (Lloyd / Yinyang tables; the k-NN tables have their own
// kernels).  As separate kernels it would be ten stream operations (three memsets, ||c||^2, mean, mu, centred norms,
// maximum, scale, table) of 3-12 us each on a 1 MB centroid matrix: ~0.05 ms of dependent launches per pass, 1 % of the
// step of an 8M-row shard and 8 % of the step of a 1M-row shard (8 GPUs).  Here they run as four phases of one small
// grid separated by a sense-reversing grid barrier; every CTA is resident (grid <= number of SMs, 256 threads, 38 KB
// static shared memory), so the barrier cannot deadlock.  Values produced by other CTAs in an earlier phase are read
// with ld.global.cg.
// ---------------------------------------------------------------------------------------------------
struct PrepArgs {
  int metric, D, nkb, by_source;
  uint32_t K, rows_pad;
  const float* C;
  float* csq;            // reference-order ||c||^2 (L2) / 1 (cosine); written here when compute_csq
  int compute_csq;
  float* cnorm2;         // L2: ||c - mu||^2; cosine: upper bound of ||c||^2
  double* musum;         // [D] + valid-row count
  float* neg_mu_s;       // [nkb * KB]
  Stats* stats;
  uint32_t* counters;    // CNT_N words, zeroed here
  __half* table;
  __half* aug_blob;
  const uint32_t* gather;
  unsigned* barrier;     // {arrivals, generation}
};

__device__ __forceinline__ void prep_grid_barrier(unsigned* bar, unsigned nblocks) {
  __syncthreads();
  if (threadIdx.x == 0) {
    volatile unsigned* gen = bar + 1;
    const unsigned g = *gen;          // cannot advance before this CTA has arrived
    __threadfence();
    if (atomicAdd(bar, 1u) == nblocks - 1u) {
      atomicExch(bar, 0u);
      __threadfence();
      atomicAdd(bar + 1, 1u);
    } else {
      while (*gen == g) __nanosleep(32);
    }
    __threadfence();
  }
  __syncthreads();
}

__global__ void __launch_bounds__(256)
tc_prep_fused_kernel(const PrepArgs a) {
  __shared__ float s_tile[8][32 * 33];   // ||c||^2: one 32 x 32 staging tile per warp
  __shared__ float s_mu[MAX_TILE64_NKB * KB];
  __shared__ float s_scale;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const uint32_t gw = blockIdx.x * 8u + warp, nw = gridDim.x * 8u;
  const uint32_t gt = blockIdx.x * 256u + tid, nthr = gridDim.x * 256u;
  const int D = a.D;
  const uint32_t K = a.K;

  // ---- phase 0: zero the pass counters / statistics / column sums; ||c||^2 in the reference's order
  if (gt < CNT_N) a.counters[gt] = 0u;
  if (gt < sizeof(Stats) / 4) reinterpret_cast<uint32_t*>(a.stats)[gt] = 0u;
  if (a.metric == 0)
    for (uint32_t i = gt; i < static_cast<uint32_t>(D) + 1u; i += nthr) a.musum[i] = 0.0;
  if (a.compute_csq) {
    float* tile = s_tile[warp];
    for (uint32_t c0 = gw * 32u; c0 < K; c0 += nw * 32u) {
      if (a.metric == 1) {
        if (c0 + lane < K) a.csq[c0 + lane] = 1.f;
        continue;
      }
      // lane r walks row c0 + r in feature order (the reference's sequential Kahan sum); 32 features x 32 rows are
      // staged through shared memory with coalesced loads (lane = feature), and the loads of the NEXT 32 features are
      // in flight during the walk -- this phase is the longest of the launch (a 256-step dependent chain per row)
      kmb::Kahan k;
      float v[32];
      auto load32 = [&](int f0) {
        const int fl = min(32, D - f0);
#pragma unroll
        for (int r = 0; r < 32; r++) {
          const uint32_t c = min(c0 + r, K - 1);
          v[r] = lane < fl ? a.C[static_cast<size_t>(c) * D + f0 + lane] : 0.f;
        }
      };
      load32(0);
      for (int f0 = 0; f0 < D; f0 += 32) {
        const int fl = min(32, D - f0);
#pragma unroll
        for (int r = 0; r < 32; r++) tile[r * 33 + lane] = v[r];
        __syncwarp();
        if (f0 + 32 < D) load32(f0 + 32);
        for (int f = 0; f < fl; f++) {
          const float x = tile[lane * 33 + f];
          k.mac(x, x);
        }
        __syncwarp();
      }
      if (c0 + lane < K) a.csq[c0 + lane] = k.sum;
    }
  }
  prep_grid_barrier(a.barrier, gridDim.x);

  const float* nsq = a.csq;
  if (a.metric == 1) {
    // ---- cosine: upper bound of ||c||^2 per centroid + its maximum
    uint32_t best = 0;
    for (uint32_t row = gw; row < K; row += nw) {
      const float* src = a.C + static_cast<size_t>(row) * D;
      float acc = 0.f;
      for (int f = lane; f < D; f += 32) {
        float v = src[f];
        acc = fmaf(v, v, acc);
      }
      for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
      const float v = acc * 1.0001f;
      if (lane == 0) a.cnorm2[row] = v;
      if (v == v && v < 3.0e38f) best = max(best, __float_as_uint(fmaxf(v, 0.f)));
    }
    if (lane == 0 && best) atomicMax(&a.stats->csq_max_bits, best);
    nsq = a.cnorm2;
    prep_grid_barrier(a.barrier, gridDim.x);
  } else {
    // ---- L2, phase 1: the centring vector mu of the filter (see Params::neg_mu_s) is the mean of the valid centroids
    // (rows whose ||c||^2 is finite).  ANY vector is a correct choice of mu (scores shift by a per-row constant); the
    // mean minimises the operand norms.  Column sums, 128 features per half CTA
    {
      const int fb = (D + 127) / 128;
      const uint32_t nvb = static_cast<uint32_t>(fb) * ((K + 15u) / 16u);   // 16 rows per half CTA: two load groups deep
      const int ht = tid & 127;
      for (uint32_t vb = blockIdx.x * 2u + (tid >> 7); vb < nvb; vb += gridDim.x * 2u) {
        const int f = static_cast<int>(vb % fb) * 128 + ht;
        const uint32_t r0 = (vb / fb) * 16u, r1 = min(K, r0 + 16u);
        double acc = 0.0;
        uint32_t nv = 0;
        for (uint32_t rb = r0; rb < r1; rb += 8) {
          float v[8], q[8];
#pragma unroll
          for (int j = 0; j < 8; j++) {
            const uint32_t r = min(rb + j, r1 - 1);
            q[j] = __ldcg(a.csq + r);
            v[j] = f < D ? a.C[static_cast<size_t>(r) * D + f] : 0.f;
          }
#pragma unroll
          for (int j = 0; j < 8; j++) {
            if (rb + j >= r1 || !(q[j] == q[j] && q[j] < 3.0e38f)) continue;
            nv++;
            acc += static_cast<double>(v[j]);
          }
        }
        if (f < D && nv) atomicAdd(&a.musum[f], acc);
        if (vb % fb == 0 && ht == 0 && nv) atomicAdd(reinterpret_cast<uint32_t*>(a.musum + D), nv);
      }
    }
    prep_grid_barrier(a.barrier, gridDim.x);
    // ---- phase 2: mu (every CTA keeps its own copy), ||c - mu||^2 per centroid, its maximum
    {
      const uint32_t nv = __ldcg(reinterpret_cast<const uint32_t*>(a.musum + D));
      for (int f = tid; f < D; f += 256) {
        const float m = nv ? static_cast<float>(__ldcg(a.musum + f) / nv) : 0.f;
        const float mm = (fabsf(m) < 3.0e38f) ? m : 0.f;
        s_mu[f] = mm;
      }
      __syncthreads();
      uint32_t best = 0;
      for (uint32_t row = gw; row < K; row += nw) {
        const float* src = a.C + static_cast<size_t>(row) * D;
        double acc = 0.0;
        for (int f = lane; f < D; f += 32) {
          const float v = src[f] - s_mu[f];
          acc += static_cast<double>(v) * v;
        }
        for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
        const float q = __ldcg(a.csq + row);
        const float v = (q == q && q < 3.0e38f) ? static_cast<float>(acc) : q;   // dead centroids stay dead
        if (lane == 0) a.cnorm2[row] = v;
        if (v == v && v < 3.0e38f) best = max(best, __float_as_uint(fmaxf(v, 0.f)));
      }
      if (lane == 0 && best) atomicMax(&a.stats->csq_max_bits, best);
    }
    nsq = a.cnorm2;
    prep_grid_barrier(a.barrier, gridDim.x);
  }

  // ---- phase 3: scale (every CTA derives it; CTA 0 publishes Stats and -mu*s), then the fp16 table + bias blocks
  const bool have_mu = a.metric == 0;
  if (warp == 0) {
    const float cmax = __fsqrt_ru(__uint_as_float(__ldcg(&a.stats->csq_max_bits)));
    const float s = prep_scale(cmax);
    if (lane == 0) s_scale = s;
    if (blockIdx.x == 0) {
      const int Dp = a.nkb * KB;
      float m2 = 0.f;
      for (int f = lane; f < Dp; f += 32) {
        const float m = (have_mu && f < D) ? s_mu[f] : 0.f;
        a.neg_mu_s[f] = -m * s;
        m2 = fmaf(m * s, m * s, m2);
      }
      for (int o = 16; o > 0; o >>= 1) m2 += __shfl_xor_sync(0xffffffffu, m2, o);
      if (lane == 0) {
        a.stats->scale = s;
        a.stats->cmax = cmax * s * 1.001f;
        // (1.002: the lane-partial sums are added in a different order than a serial loop)
        a.stats->mun = __fsqrt_ru(m2) * 1.002f;
      }
    }
  }
  __syncthreads();
  const float s = s_scale;
  for (uint32_t row = gw; row < a.rows_pad; row += nw)
    prep_table_row(row, lane, s, a.metric, a.C, nsq, K, D, a.nkb, a.table, a.aug_blob, a.stats, a.gather,
                   have_mu ? s_mu : nullptr, a.by_source);
}

// ---------------------------------------------------------------------------------------------------
// the main kernel
// ---------------------------------------------------------------------------------------------------
// bars_u32 = shared-space address of bars[0] (computed once per thread)
#define TC_WAIT(bar, parity, site) \
  ptx::mbar_wait(bars_u32 + 8u * static_cast<uint32_t>(bar), (parity), p.counters + CNT_ERR, site, bars_u32 + 8u * 63u)

// the reference's bookkeeping for one decided row (kmeans.cu:356-363); returns 1 if the assignment changed
__device__ __forceinline__ uint32_t commit_assignment(uint32_t* __restrict__ assign, uint32_t* __restrict__ prev,
                                                      uint64_t row, uint32_t winner) {
  const uint32_t a = assign[row];
  prev[row] = a;
  if (a == winner) return 0u;
  assign[row] = winner;
  return 1u;
}

// in-place compaction of one epilogue thread's list: an entry whose chunk maxima of both rows fell below their rows'
// current thresholds can never hold a candidate (the thresholds only rise)
__device__ __forceinline__ uint32_t compact_list(uint32_t* lst, uint16_t* lnt, uint32_t cnt, float thr0, float thr1) {
  // lst / lnt = this thread's column of the entry arrays / of the n-tiles (stride 256 per entry, LIST_ARRAY bytes
  // between arrays)
  constexpr uint32_t A = LIST_ARRAY / 4;
  uint32_t w = 0;
#pragma unroll 1
  for (uint32_t i = 0; i < cnt; i++) {
    if (__uint_as_float(lst[i * 256]) >= thr0 || __uint_as_float(lst[A + i * 256]) >= thr1) {
      if (w != i) {
        for (int k = 0; k < LIST_ARRAYS; k++) lst[k * A + w * 256] = lst[k * A + i * 256];
        lnt[w * 256] = lnt[i * 256];
      }
      w++;
    }
  }
  return w;
}

// MODE 2: the n-tiles query tile `tile` is multiplied with, 0 = nothing to do.  T64: tile t is half t & 1 of table
// block t >> 1 (the per-block arrays are read there); a half without live rows has nothing to do
template <bool T64>
__device__ __forceinline__ uint32_t knn_tile_nblk(const Params& p, uint32_t tile) {
  if (!T64) return p.knn_nblk[tile];
  return (tile & 1u) * 64u < p.tile_nrows[tile >> 1] ? p.knn_nblk[tile >> 1] : 0u;
}

// enumerates the n-tiles (blocks of 128 table rows) one sample tile is multiplied with, segment by segment
// (MODE 0 / 1: one segment = the whole table; MODE 2: one segment per candidate cluster)
template <int MODE, bool T64 = false>
struct BlockIter {
  uint32_t cur, lo, hi, left;    // current block, bounds of the current segment, blocks left including cur
  const uint2* rg;
  __device__ __forceinline__ BlockIter(const Params& p, uint32_t tile) {
    if (MODE == 2) {
      left = knn_tile_nblk<T64>(p, tile);
      rg = p.knn_ranges + p.knn_roff[T64 ? tile >> 1 : tile];
      if (left) { lo = cur = rg->x; hi = rg->y; } else { lo = cur = hi = 0; }
    } else {
      left = static_cast<uint32_t>(p.nt);
      lo = cur = 0;
      hi = left - 1;
      rg = nullptr;
    }
  }
  __device__ __forceinline__ bool valid() const { return left != 0; }
  __device__ __forceinline__ bool seg_first() const { return cur == lo; }
  __device__ __forceinline__ bool seg_last() const { return cur == hi; }
  __device__ __forceinline__ void next() {
    left--;
    if (MODE != 2) { cur++; return; }   // (keeps the range-list load out of the Lloyd / Yinyang loops: measured 0.65 ms per pass)
    if (cur == hi && left) { rg++; lo = cur = rg->x; hi = rg->y; } else { cur++; }
  }
};

// k-NN epilogue helpers (rare paths, kept out of line): sorted insert into the half-row's descending top-kk column
// in shared memory; returns the new kk-th largest value
__device__ __noinline__ float knn_topk_insert(float* col, int kk, float v) {
  int j = kk - 1;
  while (j > 0 && col[(j - 1) * 256] < v) {
    col[j * 256] = col[(j - 1) * 256];
    j--;
  }
  col[j * 256] = v;
  return col[(kk - 1) * 256];
}
// threshold sweep of the k-NN pass: every half-row keeps 32 running maxima over disjoint column buckets (branch
// free); afterwards the kk largest of the row's 64 buckets (both halves) become the descending top-kk list
__device__ __noinline__ void knn_select_buckets(const float* mine, const float* partner, int kk, float goff,
                                                float* out) {
  unsigned long long taken = 0ull;
  for (int o = 0; o < kk; o++) {
    float best = -INFINITY;
    int bi = -1;
    for (int j = 0; j < 64; j++) {
      const float v = j < 32 ? mine[j * 256] : partner[(j - 32) * 256];
      if (!((taken >> j) & 1ull) && v > best) { best = v; bi = j; }
    }
    if (bi >= 0) taken |= 1ull << bi;
    out[o] = best - goff;
  }
}
// the same at 64-row tiles: the kk largest of the row's 128 buckets, 32 in each of its four parts (b = bucket 0 of part
// 0; part q is TR = 64 columns of the scratch further on)
__device__ __noinline__ void knn_select_buckets4(const float* b, int kk, float goff, float* out) {
  unsigned long long taken0 = 0ull, taken1 = 0ull;   // parts 0-1 | parts 2-3
  for (int o = 0; o < kk; o++) {
    float best = -INFINITY;
    int bi = -1;
#pragma unroll
    for (int q = 0; q < 4; q++) {
      const unsigned long long tk = q < 2 ? taken0 : taken1;
      for (int j = 0; j < 32; j++) {
        const float v = b[q * 64 + j * 256];
        if (!((tk >> ((q & 1) * 32 + j)) & 1ull) && v > best) { best = v; bi = q * 32 + j; }
      }
    }
    if (bi >= 64) taken1 |= 1ull << (bi - 64);
    else if (bi >= 0) taken0 |= 1ull << bi;
    out[o] = best - goff;
  }
}
// append to the half-row's global entry list; when full, drop the entries that fell below the current kk-th
// best minus their own margin (g-space)
__device__ __noinline__ uint32_t knn_append(uint4* ent, uint32_t cnt, float kth, float cm, uint32_t mask, uint32_t cid,
                                            float margin, uint32_t* flags) {
  if (cnt == KNN_CAP) {
    uint32_t w = 0;
    for (uint32_t i = 0; i < cnt; i++) {
      const uint4 e = ent[i];
      if (__uint_as_float(e.x) >= kth - __uint_as_float(e.w)) ent[w++] = e;
    }
    cnt = w;
    if (cnt == KNN_CAP) { *flags |= 2u; return cnt; }
  }
  ent[cnt] = make_uint4(__float_as_uint(cm), mask, cid, __float_as_uint(margin));
  return cnt + 1;
}

// MODE 2 / 3 only (their epilogues take maxima over 4 consecutive columns and fold group runs of a 64-column half).
// Regrouping of one warp's m64n128 accumulator fragment without shared memory: acc[j*4 + hh*2 + e] is (row
// hh*8 + lane/4, column 8j + 2t + e) with t = lane % 4.  The four lanes of a quad hold the same two rows; lane t takes
// combination c = t of (row hh = c % 2, half c / 2) and receives its 16 columns from each quad partner s (columns
// 8jj + 2s + e of the half, jj = 0..7) in three xor rounds.  r0 / r1 = columns 0-31 / 32-63 of the half.
__device__ __forceinline__ void regroup_quad(const float (&acc)[64], int lane, uint32_t (&r0)[32], uint32_t (&r1)[32]) {
  const int t = lane & 3;
#pragma unroll
  for (int jj = 0; jj < 8; jj++)
#pragma unroll
    for (int e2 = 0; e2 < 2; e2++) {
      // block value of combination c at (jj, e2): acc[((c / 2) * 8 + jj) * 4 + (c % 2) * 2 + e2]
      const float b00 = acc[jj * 4 + e2], b10 = acc[jj * 4 + 2 + e2];
      const float b01 = acc[(8 + jj) * 4 + e2], b11 = acc[(8 + jj) * 4 + 2 + e2];
      float got[4];   // got[k]: from partner t ^ k, column 8jj + 2 (t ^ k) + e2 of this lane's (row, half)
#pragma unroll
      for (int k = 0; k < 4; k++) {
        const int c = t ^ k;                     // the partner's combination: what it needs from this lane
        const float v = (c & 2) ? ((c & 1) ? b11 : b01) : ((c & 1) ? b10 : b00);
        got[k] = k ? __shfl_xor_sync(0xffffffffu, v, k) : v;
      }
#pragma unroll
      for (int s = 0; s < 4; s++) {
        const int k = s ^ t;
        const float v = (k & 2) ? ((k & 1) ? got[3] : got[2]) : ((k & 1) ? got[1] : got[0]);
        const int col = 8 * jj + 2 * s + e2;     // 0..63 within the half
        (col < 32 ? r0[col] : r1[col - 32]) = __float_as_uint(v);
      }
    }
}
// MODE 2 at 64-row tiles: the same for one warp's m64n64 fragment, acc[j*4 + hh*2 + e] = (row hh*8 + lane/4, column
// 8j + 2t + e of the warpgroup's 64-column half), j < 8.  Lane t takes combination c = t of (row hh = c % 2, quarter
// c / 2) and receives its columns 8jj + 2s + e (jj = 0..3) of the quarter from each quad partner s: r = the quarter's
// 32 consecutive columns.
__device__ __forceinline__ void regroup_quad_t64(const float (&acc)[32], int lane, uint32_t (&r)[32]) {
  const int t = lane & 3;
#pragma unroll
  for (int jj = 0; jj < 4; jj++)
#pragma unroll
    for (int e2 = 0; e2 < 2; e2++) {
      // block value of combination c at (jj, e2): acc[((c / 2) * 4 + jj) * 4 + (c % 2) * 2 + e2]
      const float b00 = acc[jj * 4 + e2], b10 = acc[jj * 4 + 2 + e2];
      const float b01 = acc[(4 + jj) * 4 + e2], b11 = acc[(4 + jj) * 4 + 2 + e2];
      float got[4];
#pragma unroll
      for (int k = 0; k < 4; k++) {
        const int c = t ^ k;
        const float v = (c & 2) ? ((c & 1) ? b11 : b01) : ((c & 1) ? b10 : b00);
        got[k] = k ? __shfl_xor_sync(0xffffffffu, v, k) : v;
      }
#pragma unroll
      for (int s = 0; s < 4; s++) {
        const int k = s ^ t;
        const float v = (k & 2) ? ((k & 1) ? got[3] : got[2]) : ((k & 1) ? got[1] : got[0]);
        r[8 * jj + 2 * s + e2] = __float_as_uint(v);
      }
    }
}

// MODE 3: folds one row's NQ consecutive quad maxima qm (table quads with group ids gq) into per-group maxima and
// turns every finished run into a lower bound of the distance to the nearest centroid of that group, merged into
// yb[g] with an atomic minimum.  A group's run may continue in the other lanes, warpgroups or n-tiles of the row: each
// piece flushes its own bound, and since the bound never increases with the maximum, the smallest of them is the bound
// of the group's true maximum.  Eb >= E (the row's score error), xa2lo = lower bound of |s (x - mu)|^2.
template <int NQ>
__device__ __forceinline__ void yy_fold_groups(const Params& p, const float (&qm)[NQ], const uint32_t (&gq)[NQ],
                                               bool emit_ok, uint32_t gown, float Eb, float xa2lo, uint32_t* yb) {
  const float sc = p.stats->scale;
  const float inv_s = 1.f / sc, inv_s2 = inv_s * inv_s;   // s is a power of two: exact
  float run = qm[0];
#pragma unroll
  for (int i = 1; i <= NQ; i++) {
    if (i == NQ || gq[i] != gq[i - 1]) {
      const uint32_t g = gq[i - 1];
      if (emit_ok && g < p.G && g != gown) {
        float v;
        if (p.metric == 1) {
          // angular: every dot of the group <= (run + E) / s^2; acos is decreasing; libdevice acosf is good to 2 ulp
          const float dot = fminf(1.f, fmaxf(-1.f, (run + Eb) * inv_s2));
          v = fmaxf(0.f, acosf(dot) - 4.0e-6f);
        } else {
          // L2: s^2 d^2 = |x^|^2 - 2 score  >=  |x^|^2 - 2 (run + E)
          const float t = xa2lo - 2.f * (run + Eb);
          v = t > 0.f ? __fsqrt_rd(t) * inv_s * (1.f - 4.0e-6f) : 0.f;
        }
        atomicMin(yb + g, __float_as_uint(v));        // bounds are >= +0: ordered like unsigned integers
      }
      if (i < NQ) run = qm[i];
    } else {
      run = fmaxf(run, qm[i]);
    }
  }
}

// NKB: K-blocks of 64 features (compile-time: the MMA issue loop must be branch- and address-arithmetic-free); MODE 0 =
// Lloyd assignment, 1 = Yinyang local step, 2 = k-NN, 3 = Yinyang bounds refresh (see Params); the kernels below wrap
// it as tc_assign_kernel<NKB, MODE> and tc_assign_rows_kernel<NKB>.  ROWS (MODE 0 only): the
// mini-batch pass over a row list -- position i of the pass is sample p.rows[i]: the converters load X[rows[i]], results
// and the re-check queue are by position (pair_row keeps the sample row for the re-check's loads), and a row the filter
// cannot bound goes to the overflow list as its sample row with result[i] = kOverflowRow (tc_assign_rows resolves it).
template <int NKB, int MODE, bool ROWS>
__device__ __forceinline__ void
tc_assign_body(const CUtensorMap& tmap_b, const Params& p) {
  static_assert(NKB <= MAX_TILE64_NKB, "the A operand of a tile must fit its shared-memory region");
  constexpr int BST = b_stages(NKB), AUGB = aug_bufs(NKB), NDEPTH = norm_depth(NKB), ASLOTS = a_slots(NKB);
  // NKB 9..16 (T64): 64-row tiles; consumer warpgroup g holds all 64 rows at columns 64g .. 64g + 63 of every n-tile
  constexpr bool T64 = tile64(NKB);
  constexpr int TR = tile_rows(NKB), AKB = a_kb_bytes(NKB);
  constexpr int NACC = T64 ? 32 : 64;   // accumulators per consumer thread: 2 rows x NACC / 2 columns
  // 1024-byte alignment (128B-swizzle atoms) by an OFFSET into the shared array: the pointer keeps its shared address
  // space, so every access below is LDS / STS
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (ptx::smem_u32(smem_raw) & 1023u)) & 1023u);
  const SmemLayout L = smem_layout(NKB);
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + L.bars);
  const uint32_t bars_u32 = ptx::smem_u32(bars);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  constexpr int nkb = NKB;
  // The error bound needs |x~| (the fp16-rounded operand row) and the rounding residual |a - x~|; the converters MEASURE
  // both.  (row_margin keeps the analytic bound from |a|^2 alone behind this constant: dropping that dead branch too
  // changes ptxas's instruction schedule of tc_assign_kernel<1..8, 1>.)
  constexpr bool MEASURED_RESIDUAL = true;
  [[maybe_unused]] const int nt = p.nt;
  const uint32_t n_eff = MODE == 1 ? min(*p.d_nrows, p.n) : p.n;
  constexpr uint32_t KNN_TPB = T64 ? 2u : 1u;   // MODE 2: query tiles per 128-row table block
  const uint32_t ntiles = MODE == 1 ? (n_eff + TR - 1) / TR : (MODE == 2 ? *p.d_ntiles * KNN_TPB : p.ntiles);
  // MODE 2 on several GPUs: this device serves the query tiles of part knn_part of knn_nparts (every GPU holds the
  // whole candidate table; tiles are independent).  The shards are whole blocks, as in range_build_kernel and
  // expand_kernel.
  uint32_t tile_lo = 0, tile_end = ntiles;
  if (MODE == 2 && p.knn_nparts > 1) {
    const uint32_t nblk = ntiles / KNN_TPB;
    tile_lo = static_cast<uint32_t>(static_cast<uint64_t>(nblk) * p.knn_part / p.knn_nparts) * KNN_TPB;
    tile_end = static_cast<uint32_t>(static_cast<uint64_t>(nblk) * (p.knn_part + 1) / p.knn_nparts) * KNN_TPB;
  }
  const uint32_t tile_begin = tile_lo + blockIdx.x;

  if (warp == WARP_B_PRODUCER && lane == 0) {
    bars[63] = 0ull;   // "a wait has given up" flag (mbar_wait_slow)
    ptx::prefetch_tmap(&tmap_b);
    // every consumer warp releases the shared-memory operands it has read, once its own wgmma.wait_group returned
    for (int s = 0; s < BST; s++) {
      ptx::mbar_init(&bars[BAR_B_FULL + s], 1);
      ptx::mbar_init(&bars[BAR_B_EMPTY + s], N_EPI_WARPS);
    }
    for (int s = 0; s < 2; s++) {
      ptx::mbar_init(&bars[BAR_AUG_FULL + s], 1);
      ptx::mbar_init(&bars[BAR_AUG_EMPTY + s], N_EPI_WARPS);
      ptx::mbar_init(&bars[BAR_EMIT_FULL + s], N_EPI_WARPS);
      ptx::mbar_init(&bars[BAR_EMIT_EMPTY + s], N_EMIT_WARPS);
    }
    for (int s = 0; s < ASLOTS; s++) {
      ptx::mbar_init(&bars[BAR_A_FULL + s], N_CONV_WARPS);
      ptx::mbar_init(&bars[BAR_A_FREE + s], N_EPI_WARPS);
    }
    ptx::fence_mbar_init();
  }
  // constant A-side bias block: ones in the first three K positions of every row
  for (int i = threadIdx.x; i < TR * 16; i += N_THREADS) {
    int r = i >> 4, k = i & 15;
    int j = k >> 3, e = k & 7;
    reinterpret_cast<__half*>(smem + L.aug_a)[(j * (TR * 16) + (r >> 3) * 128 + (r & 7) * 16) / 2 + e] =
        __float2half_rn(k < 3 ? 1.f : 0.f);
  }
  for (int i = threadIdx.x; i < mu_features(NKB); i += N_THREADS)
    reinterpret_cast<float*>(smem + L.mu)[i] = (MODE != 2 && p.neg_mu_s && i < nkb * KB) ? p.neg_mu_s[i] : 0.f;
  ptx::fence_proxy_async_smem();
  __syncthreads();

  // Role dispatch.  setmaxnreg is executed once by every warp of a warpgroup, at the top of the warpgroup's branch
  // (there ptxas allocates the branch within the new count).
  if (warp < FIRST_CONV_WARP) {
    ptx::setmaxnreg_dec<REGS_WG0>();
    if (warp == WARP_B_PRODUCER) {
      // ================================ TMA producer: centroid table + bias blocks ================================
      if (lane == 0) {
        uint32_t bs = 0, bph = 0, ac = 0;      // B ring stage / phase, bias blocks issued
        for (uint32_t tile = tile_begin; tile < tile_end; tile += gridDim.x) {
          for (BlockIter<MODE, T64> it(p, tile); it.valid(); it.next()) {
            const int n = static_cast<int>(it.cur);
#pragma unroll
            for (int kb = 0; kb < NKB; kb++) {
              TC_WAIT(BAR_B_EMPTY + bs, bph ^ 1, 1);
#if KMB_KO == 5
              ptx::mbar_arrive(&bars[BAR_B_FULL + bs]);
#else
              ptx::mbar_arrive_expect_tx(&bars[BAR_B_FULL + bs], B_KB_BYTES);
              ptx::tma_load_2d(smem + L.b + bs * B_STAGE_BYTES, &tmap_b, kb * KB, n * TN, &bars[BAR_B_FULL + bs]);
#endif
              if (++bs == BST) { bs = 0; bph ^= 1; }
            }
            // the bias block after the K-blocks: it is consumed last, and with one buffer its release (the end of the
            // previous n-tile) must not hold back the centroid stages of this one
            const int as = ac % AUGB;
            const uint32_t aph = (ac / AUGB) & 1;
            TC_WAIT(BAR_AUG_EMPTY + as, aph ^ 1, 2);
#if KMB_KO == 5
            ptx::mbar_arrive(&bars[BAR_AUG_FULL + as]);
#else
            ptx::mbar_arrive_expect_tx(&bars[BAR_AUG_FULL + as], AUG_B_BYTES);
            ptx::bulk_load(smem + L.aug_b + as * AUG_B_BYTES,
                           reinterpret_cast<const uint8_t*>(p.aug_blob) + static_cast<size_t>(n) * AUG_B_BYTES,
                           AUG_B_BYTES, &bars[BAR_AUG_FULL + as]);
#endif
            ac++;
          }
        }
      }
    } else if (MODE < 2) {
      // ================================ emitters: merge column halves, write results / queues ================================
      // three warps walk the tile's 128 rows with a stride of 96: warp 0 takes two rows per thread
      // (T64: rows 64 and up are not live, so only warps 0 and 1 emit rows; every warp still takes part in the queue
      // reservation and the release)
      const int row0 = (warp - FIRST_EMIT_WARP) * 32 + lane;
      const int nrows = row0 + N_EMIT_WARPS * 32 < TM ? 2 : 1;   // warp-uniform
      const float cap = p.metric == 1 ? p.stats->scale * p.stats->scale : INFINITY;
      const uint32_t force = p.stats->force_exact ? 16u : 0u;
      uint32_t ti = 0, nchanged = 0;
      for (uint32_t tile = tile_begin; tile < tile_end; tile += gridDim.x, ti++) {
        const int par = ti & 1;
        const uint32_t* lst = reinterpret_cast<const uint32_t*>(smem + L.list) + par * LIST_LEN * 256;
        const uint16_t* lnt = reinterpret_cast<const uint16_t*>(smem + L.list + LIST_ARRAYS * LIST_ARRAY) + par * LIST_LEN * 256;
        const float* fin = reinterpret_cast<const float*>(smem + L.fin) + par * FIN_WORDS;
        const uint32_t* finu = reinterpret_cast<const uint32_t*>(fin);
        TC_WAIT(BAR_EMIT_FULL + par, (ti >> 1) & 1, 12);
        for (int ri = 0; ri < nrows; ri++) {
          const int row = row0 + ri * N_EMIT_WARPS * 32;
          uint64_t grow = static_cast<uint64_t>(tile) * TR + row;
          uint32_t cand[MAX_CAND];
          uint32_t total = 0, fl = 0;
          const bool live = (!T64 || row < TR) && grow < n_eff;
          if (MODE == 1 && live) grow = p.rows[grow];
          if (live) {
            // the row's four epilogue threads: lanes 4 (row % 8) + t of consumer warp row / 16; the row is their R0 or R1
            // (T64: eight threads, the same four lanes in both warpgroups, 128 list columns apart)
            const int hh = (row >> 3) & 1;
            const int lid0 = (row >> 4) * 32 + (row & 7) * 4;
            // MODE 1: the second largest of the row's chunk maxima (a lower bound of its second best score).  T64: each
            // warpgroup's maximum covers its own columns only, so each is <= the row maximum and every warpgroup's
            // candidate set contains the one of the row maximum; the final threshold uses the larger of the two.
            float Mf;
            if constexpr (T64 && MODE == 1) {
              // T64, MODE 1: warpgroup g keeps its own pair (M1_g, M2_g) over its 64 columns of every n-tile.  Two
              // distinct columns reach each M2_g, and M1_0 / M1_1 come from disjoint columns, so the row's second best
              // score is >= max(M2_0, M2_1, min(M1_0, M1_1)) (DESIGN §4k).  The MODE 0 merge max(M2_0, M1_1) is not a
              // lower bound: M1_1 may be the row's best score.
              Mf = ptx::fmax3(fin[FIN_M2 + row], fin[FIN_M2 + TR + row], fminf(fin[FIN_M + row], fin[FIN_M + TR + row]));
            } else {
              Mf = MODE == 1 ? fin[FIN_M2 + row] : fin[FIN_M + row];
              if (T64) Mf = fmaxf(Mf, fin[FIN_M + TR + row]);
            }
            const float mg = fin[FIN_MARGIN + row];
            const float thr = fminf(Mf, cap) - mg;
            fl = force;
            // cosine: if every dot may be <= -1 they all clamp to pi and the lowest index wins -> exact pass
            if (p.metric == 1 && !(Mf >= mg - cap)) fl |= 8u;
            // padded table rows and dead (non-finite) centroids score exactly -65504 (zero row + sentinel bias): a
            // threshold that low cannot tell them from real candidates (an outlier far from every centroid) -> exact pass
            if (!(thr > SENTINEL_GUARD)) fl |= 8u;
            // Candidates reach cand[] ordered by (lane, entry, bit), not by column.  Nothing downstream depends on that
            // order: the re-check reduction picks the smallest index among equal scores (sc == best && c < arg), and the
            // Yinyang finish takes a warp minimum of the index.
            for (int t = 0; t < (T64 ? 8 : 4); t++) {
              const int tq = T64 ? t & 3 : t, wg = T64 ? t >> 2 : 0;
              const int sl = lid0 + wg * 128 + tq;
              const uint32_t st = finu[FIN_STATE + sl];
              fl |= (st >> (8 + 8 * hh)) & 0xffu;
              const uint32_t c2 = st & 0xffu;
              for (uint32_t i = 0; i < c2; i++) {
                constexpr uint32_t A = LIST_ARRAY / 4;
                if (!(__uint_as_float(lst[hh * A + i * 256 + sl]) >= thr)) continue;   // the row's chunk maximum
                const uint32_t base = static_cast<uint32_t>(lnt[i * 256 + sl]) * TN + 64 * wg + 2 * tq;
                uint32_t m = lst[(2 + hh) * A + i * 256 + sl];
                while (m) {
                  const int b = __ffs(m) - 1;
                  m &= m - 1;
                  // bit b = 2j + e: column 8j + 2t + e (T64: 16-bit masks, j < 8, of the warpgroup's 64-column half)
                  const uint32_t col = base + 8 * (b >> 1) + (b & 1);
                  if (col < p.K) {
                    if (total < MAX_CAND) cand[total] = col;
                    total++;
                  }
                }
              }
            }
          }
          // the lists of this parity are consumed once the warp's last row has read them: the epilogue may start tile ti+2
          if (ri == nrows - 1) {
            __syncwarp();
            if (lane == 0) ptx::mbar_arrive(&bars[BAR_EMIT_EMPTY + par]);
          }
          const bool overflow = live && (fl || total > MAX_CAND || (MODE == 1 && total == 0));
          const bool multi = live && !overflow && total >= (MODE == 1 ? 1u : 2u);
          // warp-aggregated queue reservation: one atomic per warp for the pairs, one for the row queue
          uint32_t want = multi ? total : 0, pre = want;
#pragma unroll
          for (int o = 1; o < 32; o <<= 1) {
            uint32_t v = __shfl_up_sync(0xffffffffu, pre, o);
            if (lane >= o) pre += v;
          }
          const uint32_t warp_total = __shfl_sync(0xffffffffu, pre, 31);
          const unsigned mmask = __ballot_sync(0xffffffffu, multi);
          uint32_t base = 0, rqbase = 0;
          if (lane == 0 && warp_total) {
            base = atomicAdd(&p.counters[CNT_PAIRS], warp_total);
            rqbase = atomicAdd(&p.counters[CNT_ROWQ], static_cast<uint32_t>(__popc(mmask)));
          }
          base = __shfl_sync(0xffffffffu, base, 0) + (pre - want);
          rqbase = __shfl_sync(0xffffffffu, rqbase, 0) + __popc(mmask & ((1u << lane) - 1));
          if (live) {
            if (overflow) {
              p.ovf_rows[atomicAdd(&p.counters[CNT_OVF], 1u)] = ROWS ? p.rows[grow] : static_cast<uint32_t>(grow);
              if (ROWS) p.result[grow] = kOverflowRow;
            } else if (MODE == 0 && total == 1) {
              if (p.assign) nchanged += commit_assignment(p.assign, p.prev, grow, cand[0]);
              else p.result[grow] = cand[0];
            } else if (MODE == 0 && total == 0) {
              // every score NaN: nothing wins, the assignment stays (reference kmeans.cu:349-353)
              if (!p.assign) p.result[grow] = kUntouched;
            } else if (base + total <= p.max_pairs) {
              for (uint32_t i = 0; i < total; i++) {
                p.pair_row[base + i] = ROWS ? p.rows[grow] : static_cast<uint32_t>(grow);
                p.pair_cand[base + i] = cand[i];
              }
              p.rowq[3 * rqbase] = static_cast<uint32_t>(grow);
              p.rowq[3 * rqbase + 1] = base;
              p.rowq[3 * rqbase + 2] = total;
            } else {
              // queue full: the row goes to the full exact pass; its reserved row-queue slot is neutralised
              p.rowq[3 * rqbase] = static_cast<uint32_t>(grow);
              p.rowq[3 * rqbase + 1] = 0;
              p.rowq[3 * rqbase + 2] = 0;
              p.ovf_rows[atomicAdd(&p.counters[CNT_OVF], 1u)] = ROWS ? p.rows[grow] : static_cast<uint32_t>(grow);
              if (ROWS) p.result[grow] = kOverflowRow;
            }
          }
        }
      }
      if (MODE == 0 && p.assign) {
        nchanged = __reduce_add_sync(0xffffffffu, nchanged);
        if (lane == 0 && nchanged) atomicAdd(p.d_changed, nchanged);
      }
    }
  } else if (warp >= FIRST_CONV_WARP && warp < FIRST_CONV_WARP + N_CONV_WARPS) {
    ptx::setmaxnreg_dec<REGS_CONV>();
    // ================================ converters: fp32 rows -> fp16 A operand in shared memory ================================
    const int q = warp & 3;
    // this thread's sample row within the tile; T64: two threads per row, each converting one half of every K-block
    const int row = T64 ? q * 16 + (lane >> 1) : q * 32 + lane;
    const int hsel = T64 ? lane & 1 : 0;
    const float s = p.stats->scale;
    uint32_t si = 0, as = 0, aph = 0;       // segments converted; A ring slot and phase of the next K-block
    for (uint32_t tile = tile_begin; tile < tile_end; tile += gridDim.x) {
      if (MODE == 2 && knn_tile_nblk<T64>(p, tile) == 0) continue;
      const float* xrow = nullptr;
      bool xlive = true;                      // rows past the end of the samples convert as zeros
      if (MODE == 0 || MODE == 3) {
        const uint64_t grow = static_cast<uint64_t>(tile) * TR + row;
        xlive = grow < p.n;
        xrow = p.X + (xlive ? (ROWS ? static_cast<uint64_t>(p.rows[grow]) : grow) : 0ull) * p.D;
      }
      if (MODE == 1) {
        const uint32_t li = min(tile * TR + row, n_eff - 1);   // ragged tail: repeat the last listed row
        xrow = p.X + static_cast<size_t>(p.rows[li]) * p.D;
      }
      if (MODE == 2)   // padding rows of the table repeat sample 0; they are never recorded
        xrow = p.X + static_cast<size_t>(min(p.rows[tile * TR + row], p.n - 1)) * p.D;
      const uint32_t kblk = T64 ? tile >> 1 : tile;   // MODE 2: the table block of this tile (knn_tile_nblk)
      const uint32_t nseg = MODE == 2 ? p.knn_rcount[kblk] : 1u;
      for (uint32_t seg = 0; seg < nseg; seg++, si++) {
        // ||x~||^2 and ||s(x - mu) - x~||^2 as even/odd partial sums
        uint64_t nx2 = 0ull, nd2 = 0ull;
        const uint64_t s2 = ptx::pack2(s, s);
        const float* mu = reinterpret_cast<const float*>(smem + L.mu);
        float a2 = 0.f, a2c = 0.f, nraw = 0.f;     // MODE 2: Kahan sum of the exact (x-c)^2 s^2, and s^2 (|x|+|c|)^2
        const float* crow = nullptr;
        if (MODE == 2) crow = p.C + static_cast<size_t>(p.blk_cluster[p.knn_ranges[p.knn_roff[kblk] + seg].x]) * p.D;
        for (int kb = 0; kb < nkb; kb++) {
          uint32_t pk[32];
#pragma unroll
          for (int hi = 0; hi < (T64 ? 1 : 2); hi++) {
            const int half = T64 ? hsel : hi;
            float4 gv[8];
            const int f0 = kb * KB + half * 32;
#pragma unroll
            for (int c = 0; c < 8; c++)
              gv[c] = (xlive && f0 + c * 4 < p.D) ? __ldg(reinterpret_cast<const float4*>(xrow + f0 + c * 4))
                                                  : make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
            for (int c = 0; c < (KMB_KO == 3 ? 0 : 8); c++) {
              float4 v = gv[c];
              float4 m4 = make_float4(0.f, 0.f, 0.f, 0.f);
              if (MODE == 2) {
                const float4 cv = (f0 + c * 4 < p.D) ? ptx::ldg_nc_f4(crow + f0 + c * 4) : make_float4(0.f, 0.f, 0.f, 0.f);
                const float r0 = fabsf(v.x) + fabsf(cv.x), r1 = fabsf(v.y) + fabsf(cv.y);
                const float r2 = fabsf(v.z) + fabsf(cv.z), r3 = fabsf(v.w) + fabsf(cv.w);
                nraw = fmaf(r0, r0, nraw); nraw = fmaf(r1, r1, nraw); nraw = fmaf(r2, r2, nraw); nraw = fmaf(r3, r3, nraw);
                v.x -= cv.x; v.y -= cv.y; v.z -= cv.z; v.w -= cv.w;
              } else {
                m4 = *reinterpret_cast<const float4*>(mu + f0 + c * 4);   // same address in every lane: broadcast
              }
              // a = s*v - s*mu in ONE rounding (s is a power of two, so this is exactly s * fl(v - mu))
              const uint64_t a01 = ptx::ffma2(ptx::pack2(v.x, v.y), s2, ptx::pack2(m4.x, m4.y));
              const uint64_t a23 = ptx::ffma2(ptx::pack2(v.z, v.w), s2, ptx::pack2(m4.z, m4.w));
              float a0, a1, a2_, a3;
              ptx::unpack2(a01, a0, a1);
              ptx::unpack2(a23, a2_, a3);
              __half2 h0 = __floats2half2_rn(a0, a1), h1 = __floats2half2_rn(a2_, a3);
              const float2 b0 = __half22float2(h0), b1 = __half22float2(h1);
              const uint64_t b01 = ptx::pack2(b0.x, b0.y), b23 = ptx::pack2(b1.x, b1.y);
              nx2 = ptx::ffma2(b01, b01, nx2);
              nx2 = ptx::ffma2(b23, b23, nx2);
              const uint64_t d01 = ptx::fsub2(a01, b01), d23 = ptx::fsub2(a23, b23);
              nd2 = ptx::ffma2(d01, d01, nd2);
              nd2 = ptx::ffma2(d23, d23, nd2);
              if (MODE == 2) {   // compensated: this sum is subtracted from scores of the same magnitude
                const float q4 = fmaf(a0, a0, fmaf(a1, a1, fmaf(a2_, a2_, a3 * a3)));
                const float y = q4 - a2c, t = a2 + y;
                a2c = (t - a2) - y;
                a2 = t;
              }
              pk[hi * 16 + c * 2] = *reinterpret_cast<uint32_t*>(&h0);
              pk[hi * 16 + c * 2 + 1] = *reinterpret_cast<uint32_t*>(&h1);
            }
          }
          // only the stores wait for the slot: the loads of this K-block, possibly of the next tile, are already in
          // flight while the consumers still multiply with the slot's previous K-block
          TC_WAIT(BAR_A_FREE + as, aph ^ 1, 7);
#if KMB_KO != 3
          // the row's 128 bytes of this K-block: 16-byte chunk c (features 8c .. 8c+7) at chunk position c ^ (row % 8)
          // (the 128-byte swizzle of a K-major wgmma operand; also spreads the warp's stores over all banks)
          uint8_t* a_row = smem + L.a + as * AKB + row * 128;
#pragma unroll
          for (int c = 0; c < (T64 ? 4 : 8); c++) {
            const int cc = T64 ? hsel * 4 + c : c;
            *reinterpret_cast<uint4*>(a_row + ((cc ^ (row & 7)) << 4)) =
                make_uint4(pk[4 * c], pk[4 * c + 1], pk[4 * c + 2], pk[4 * c + 3]);
          }
#else
          (void)pk;
#endif
          if (kb == nkb - 1) {
            float* norms = reinterpret_cast<float*>(smem + L.norms) + (si % NDEPTH) * 4 * TM;
            float nxl, nxh, ndl, ndh;
            ptx::unpack2(nx2, nxl, nxh);
            ptx::unpack2(nd2, ndl, ndh);
            if (T64) {   // the row's two halves (lanes 2r, 2r + 1) are combined with one 64-bit shuffle
              const uint64_t o = __shfl_xor_sync(0xffffffffu, ptx::pack2(nxl + nxh, ndl + ndh), 1);
              float onx, ond;
              ptx::unpack2(o, onx, ond);
              nxl += onx;
              ndl += ond;
              if (MODE == 2) {   // the k-NN sums too: the two compensated halves meet in one rounding (see row_margin)
                const uint64_t o2 = __shfl_xor_sync(0xffffffffu, ptx::pack2(a2, a2c), 1);
                const float onr = __shfl_xor_sync(0xffffffffu, nraw, 1);
                float oa2, oa2c;
                ptx::unpack2(o2, oa2, oa2c);
                a2 = (a2 + oa2) - (a2c + oa2c);
                nraw += onr;
              }
            }
            if (!T64 || hsel == 0) {
              norms[row] = nxl + nxh;
              norms[TM + row] = ndl + ndh;
            }
            if (MODE == 2 && (!T64 || hsel == 0)) {
              norms[2 * TM + row] = a2;
              norms[3 * TM + row] = nraw * s * s;
            }
          }
          ptx::fence_proxy_async_smem();   // the generic-proxy stores above are read by wgmma (async proxy)
          __syncwarp();
          if (lane == 0) ptx::mbar_arrive(&bars[BAR_A_FULL + as]);
          if (++as == ASLOTS) { as = 0; aph ^= 1; }
        }
      }
    }
  } else {
    ptx::setmaxnreg_inc<REGS_EPI>();
    // ================================ consumers: wgmma + epilogue ================================
    // Warpgroup g multiplies rows g*64 .. g*64+63 of the tile with all 128 columns of an n-tile; its warp wq holds the
    // accumulators of rows g*64 + wq*16 .. +15.  MODE 0 / 1 run the epilogue on that fragment as it lands: lane l holds
    // rows R0 = g*64 + wq*16 + l / 4 and R1 = R0 + 8 at columns 8j + 2t + e (t = l % 4, j < 16, e < 2), so the four
    // lanes of a quad hold all 128 columns of their two rows.  MODE 2 / 3 regroup the fragment with quad shuffles
    // first: each lane then owns one row and one 64-column half of every n-tile, lane l takes the row it already
    // holds, g*64 + wq*16 + l / 4 + 8 * (l % 2), and half (l % 4) / 2.  T64 (MODE 2 / 3): the same within warpgroup g's
    // 64-column half, so lane l holds row wq*16 + l / 4 + 8 * (l % 2) at columns 64g + 32 * ((l % 4) / 2) .. +31, part
    // 2g + (l % 4) / 2 of the row's four.
    const int e = warp - FIRST_EPI_WARP;       // 0..7
    const int g = e >> 2, wq = e & 3;
    const int h = (lane & 3) >> 1;             // MODE 2 / 3: column half of every 128-column n-tile (T64: of g's half)
    const int row = (T64 ? 0 : g * 64) + wq * 16 + (lane >> 2) + 8 * (lane & 1);
    const int kpart = T64 ? 2 * g + h : h;     // MODE 2 / 3: this thread's part of the row
    const int slot = kpart * TR + row;         // 0..255
    // T64: both warpgroups hold the same rows R0 / R1 (at columns 64g + 8j + 2t + e, j < 8) and keep their own per-row
    // maximum, MODE 1 second-best bound and margin in the per-tile state at frow = 64g + R0 (the emitters merge the two)
    const int qrow = (T64 ? 0 : g * 64) + wq * 16 + (lane >> 2);   // MODE 0 / 1: R0
    const int frow = T64 ? g * TR + qrow : qrow;
    const int lid = e * 32 + lane;                     // MODE 0 / 1: this thread's column of the lists, 0..255
    // K-major 128-byte-swizzled operands: 8-row groups 1024 bytes apart; +32 bytes (2 in the address field) per K=16.
    // T64: the whole A slot, and the 64 centroid rows (8 KiB) of this warpgroup's column half of the B stage
    const uint64_t adesc0 = ptx::make_smem_desc(ptx::smem_u32(smem + L.a + (T64 ? 0 : g * (64 * 128))), 16, 1024, 1);
    const uint64_t bdesc0 = ptx::make_smem_desc(ptx::smem_u32(smem + L.b + (T64 ? g * (64 * 128) : 0)), 16, 1024, 1);
    // bias blocks (no swizzle): core matrices of 8 rows x 16 bytes, 8-row groups 128 bytes apart, K halves TR * 16 /
    // TN * 16 bytes apart
    const uint64_t aug_ad = ptx::make_smem_desc(ptx::smem_u32(smem + L.aug_a + (T64 ? 0 : g * 1024)), TR * 16, 128, 0);
    const uint64_t aug_bd0 = ptx::make_smem_desc(ptx::smem_u32(smem + L.aug_b + (T64 ? g * 1024 : 0)), TN * 16, 128, 0);
    uint32_t bs = 0, bph = 0;                  // B ring stage / phase
    uint32_t a_ready_si = 0xFFFFFFFFu;         // segment whose A operand this warp has already waited for
    uint32_t a0 = 0, aph0 = 0;                 // A ring slot and phase of the current segment's first K-block
    // cosine: every dot >= 1 is clamped to angle 0 by the reference, so all of them tie -> the threshold
    // never rises above s^2 * 1 (the accumulator holds s^2 * dot)
    const float cap = p.metric == 1 ? p.stats->scale * p.stats->scale : INFINITY;
    uint32_t ac = 0, ti = 0, si = 0;
    for (uint32_t tile = tile_begin; tile < tile_end; tile += gridDim.x) {
      if (MODE == 2 && knn_tile_nblk<T64>(p, tile) == 0) continue;
      const int par = ti & 1;
      uint32_t* lst = reinterpret_cast<uint32_t*>(smem + L.list) + par * LIST_LEN * 256 + lid;   // this thread's entries
      uint16_t* lnt = reinterpret_cast<uint16_t*>(smem + L.list + LIST_ARRAYS * LIST_ARRAY) + par * LIST_LEN * 256 + lid;
      float* fin = reinterpret_cast<float*>(smem + L.fin) + par * FIN_WORDS;
      // the emitter warps must have consumed this parity's lists (tile ti-2)
      if (MODE < 2) TC_WAIT(BAR_EMIT_EMPTY + par, ((ti >> 1) & 1) ^ 1, 11);
      float M = -INFINITY, margin = 0.f;   // MODE 2 / 3
      // MODE 0 / 1, per row R0 / R1 (the same in the four lanes of a quad): running maximum and MODE 1 lower bound of
      // the second best score.  The rest of the state lives in fin, where the emitters read it, rather than in registers
      // across the n-tile loop: the row margins, this thread's list length and its flags (FIN_STATE).
      float Mr[2] = {-INFINITY, -INFINITY}, M2r[2] = {-INFINITY, -INFINITY};
      uint32_t* const fst = reinterpret_cast<uint32_t*>(fin) + FIN_STATE + lid;
      if (MODE < 2) *fst = 0u;
      uint32_t cnt = 0, flags = 0;       // MODE 2 / 3
      // MODE 2: this half-row's persistent state (global) and its top-kk column (the list_cm region is free)
      float* topk = reinterpret_cast<float*>(smem + L.list) + slot;   // [kk][256], kk <= 16 rows of the scratch
      uint32_t kslot = 0;
      bool klive = false;
      uint4* kent = nullptr;
      float goff = 0.f, mmax = 0.f;     // MODE 2: s^2 |x - c_B|^2 / 2 of the current segment; largest margin so far
      // MODE 3: this row's record, own group (handled exactly elsewhere), lower bound of |s (x - mu)|^2
      float xa2lo = 0.f;
      uint32_t gown = UINT32_MAX;
      uint32_t* yb = nullptr;
      bool ylive = false;
      if (MODE == 3) {
        const uint64_t grow = static_cast<uint64_t>(tile) * TR + row;
        ylive = grow < p.n;
        if (ylive) {
          const uint32_t a = p.yy_assign[grow];
          if (a < p.K) gown = p.yy_groups[a];
          yb = reinterpret_cast<uint32_t*>(p.yy_bounds + grow * (p.G + 1) + 1);
        }
      }
      uint32_t seg = 0;
      if (MODE == 2) {
        klive = static_cast<uint32_t>(T64 ? (tile & 1) * TR + row : row) < p.tile_nrows[T64 ? tile >> 1 : tile];
        kslot = (tile * TR + row) * (T64 ? 4u : 2u) + kpart;
        kent = p.knn_entries + static_cast<size_t>(kslot) * KNN_CAP;
        if (p.knn_first_pass || !klive) {
          for (int j = 0; j < p.kk; j++) topk[j * 256] = -INFINITY;
          if (p.knn_first_pass)
            for (int j = 0; j < 32; j++) topk[(16 + j) * 256] = -INFINITY;   // bucket maxima: rows 16..47 of the region
        } else {
          // second pass: every part saved the same merged list at the end of the first pass (no insertion happens
          // in the recording sweep); from here on each part adds its own, disjoint, columns
          for (int j = 0; j < p.kk; j++) topk[j * 256] = p.knn_topk[static_cast<size_t>(j) * p.knn_stride + kslot];
          cnt = p.knn_cnt[kslot];
          flags = p.knn_flags[kslot];
        }
        M = topk[(p.kk - 1) * 256];                 // MODE 2: M holds the kk-th largest group maximum (g-space)
      }
      for (BlockIter<MODE, T64> it(p, tile); it.valid(); it.next(), ac++) {
        const int n = static_cast<int>(it.cur);
        const int buf = ac % AUGB;
        const uint32_t aph = (ac / AUGB) & 1;
        const bool need_a = a_ready_si != si;      // first n-tile of this segment
        const bool free_a = it.seg_last();         // last n-tile of this segment: release each A slot once read
        a_ready_si = si;
        __syncwarp();                              // wgmma is .aligned: the warp issues it converged
        float acc[NACC];
        uint32_t sa_prev = 0;                      // A slot of the previous K-block
#pragma unroll
        for (int kb = 0; kb < NKB; kb++) {
          // K-block kb of the segment sits in slot a0 + kb of the ring (at most one wrap: NKB <= ASLOTS)
          const bool wrap = a0 + kb >= static_cast<uint32_t>(ASLOTS);
          const uint32_t sa = wrap ? a0 + kb - ASLOTS : a0 + kb;
          if (need_a) TC_WAIT(BAR_A_FULL + sa, wrap ? aph0 ^ 1 : aph0, 4);
          TC_WAIT(BAR_B_FULL + bs, bph, 5);
          __syncwarp();
#if KMB_KO != 2
          ptx::wgmma_fence_acc(acc);
          ptx::wgmma_fence();
          const uint64_t ad = adesc0 + ((sa * AKB) >> 4);
          const uint64_t bd = bdesc0 + ((bs * B_STAGE_BYTES) >> 4);
#pragma unroll
          for (int k = 0; k < 4; k++) {
            if constexpr (T64) ptx::wgmma_m64n64k16(acc, ad + 2 * k, bd + 2 * k, (kb | k) ? 1u : 0u);
            else ptx::wgmma_m64n128k16(acc, ad + 2 * k, bd + 2 * k, (kb | k) ? 1u : 0u);
          }
          ptx::wgmma_commit();
          ptx::wgmma_fence_acc(acc);
#endif
          // the previous K-block's group has retired once at most one group is pending: release its B stage (and,
          // in the segment's last n-tile, its A slot)
          if (kb > 0) {
            ptx::wgmma_wait<1>();
            if (lane == 0) {
              ptx::mbar_arrive(&bars[BAR_B_EMPTY + (bs ? bs - 1 : BST - 1)]);
              if (free_a) ptx::mbar_arrive(&bars[BAR_A_FREE + sa_prev]);
            }
          }
          sa_prev = sa;
          if (++bs == BST) { bs = 0; bph ^= 1; }
        }
        // bias step: acc += ones(64x16) * bias(128x16)^T  (both operands no-swizzle K-major smem blocks)
        TC_WAIT(BAR_AUG_FULL + buf, aph, 6);
        __syncwarp();
#if KMB_KO != 2
        ptx::wgmma_fence_acc(acc);
        ptx::wgmma_fence();
        if constexpr (T64) ptx::wgmma_m64n64k16(acc, aug_ad, aug_bd0 + buf * (AUG_B_BYTES >> 4), 1u);
        else ptx::wgmma_m64n128k16(acc, aug_ad, aug_bd0 + buf * (AUG_B_BYTES >> 4), 1u);
        ptx::wgmma_commit();
#endif
        ptx::wgmma_wait<0>();
#if KMB_KO != 2
        ptx::wgmma_fence_acc(acc);
#endif
        if (lane == 0) {
          ptx::mbar_arrive(&bars[BAR_B_EMPTY + (bs ? bs - 1 : BST - 1)]);
          ptx::mbar_arrive(&bars[BAR_AUG_EMPTY + buf]);
          if (free_a) ptx::mbar_arrive(&bars[BAR_A_FREE + sa_prev]);
        }
        if (free_a) {   // the next segment starts NKB slots further on
          a0 += NKB;
          if (a0 >= static_cast<uint32_t>(ASLOTS)) { a0 -= ASLOTS; aph0 ^= 1; }
        }
#if KMB_KO == 1
        if (MODE < 2)   // stand-in values: strictly decreasing along the row, 64 apart -> one candidate per row
#pragma unroll
          for (int j = 0; j < NACC / 4; j++)
#pragma unroll
            for (int q = 0; q < 4; q++)
              acc[j * 4 + q] = -64.f * static_cast<float>(n * TN + (T64 ? 64 * g : 0) + 8 * j + 2 * (lane & 3) + (q & 1) + 1);
#endif
        if (it.seg_first()) {
          const float* norms = reinterpret_cast<const float*>(smem + L.norms) + (si % NDEPTH) * 4 * TM;
          // (loaded here, once per segment, rather than held in registers across the n-tile loop)
          const float cmax = p.stats->cmax, dcmax = p.stats->dcmax;
          const float mun = MODE == 2 ? 0.f : p.stats->mun;
          const float knn_extra = MODE == 2 ? p.stats->knn_extra : 0.f;
          // rigorous bound on |acc - (s^2 x.c - s^2||c||^2/2)| of tile row r (see header): Cauchy-Schwarz on the
          // actual rounding residuals + accumulation + the reference's own rounding slack
          auto row_margin = [&](int r, uint32_t& fl) {
            float nx, nd;
            if (MEASURED_RESIDUAL) {
              nx = __fsqrt_ru(norms[r]) * 1.0001f;
              nd = __fsqrt_ru(norms[TM + r]) * 1.0001f;
            } else {
              // norms[r] = |a|^2 (fp32 sum, relative error < 1e-4): |a - x~| <= 2^-11 |a| + sqrt(Dp) 2^-25, |x~| <= |a| + |a - x~|
              const float na = __fsqrt_ru(norms[r]) * 1.0001f;
              nd = na * 4.8834e-4f + __fsqrt_ru(static_cast<float>(p.nkb * KB)) * 2.99e-8f;
              nx = na + nd;
              // an element beyond the fp16 range would have become Inf in the operand: such rows take the exact pass
              if (!(na < 65000.f)) fl |= 1u;
            }
            const float xn = nx + nd;
            float E = nx * dcmax + nd * cmax + nd * dcmax;
            E += static_cast<float>(p.nkb * KB + 16) * 2.4e-7f * nx * cmax;   // fp32 accumulation in the tensor core
            // reference Kahan/rd rounding + bias split + fp32 centring of both operands: the reference works on the
            // UNCENTRED vectors, whose norms are bounded by the centred ones + ||mu||
            const float xu = xn + mun, cu = cmax + mun;
            if (MODE == 0) {
              // the reference ranks with fma_rd(-2, Kahan dot, csq): |error| <= 1.2e-7 cu^2 + 2.4e-7 xu cu in score units
              // (2^-23 per directed rounding, Kahan sums to ~1 ulp); 2.5x - 5x of that is allowed for
              E += 6.0e-7f * (cu * cu + xu * cu);
            } else if (MODE == 2) {
              E += 2.0e-6f * (cu * cu + xu * cu) + 2.0e-6f * xu * xu;
            } else {
              // MODE 1 / 3 decide on TRUE distances sqrt(Kahan sum (x - c)^2): their rounding is relative to |x - c|^2 <=
              // (|x^| + |c^|)^2 (the subtraction cancels the common offset exactly), plus the fp32 centring of both operands
              E += 2.0e-6f * (xn + cmax) * (xn + cmax) + 2.4e-7f * (xn * cmax + cmax * cmax);
            }
            if (MODE == 3) {
              xa2lo = norms[r] * (1.f - 1.0e-4f);                          // lower bound of |s (x - mu)|^2 (fp32 summation error)
              // scores this low are not separable from the padding sentinel (-65504): such rows take the exact pass
              if (!(nx * cmax < 6.0e4f)) fl |= 1u;
            }
            if (MODE == 2) {
              goff = 0.5f * norms[2 * TM + r];
              // centring x - c_B and y - c_B rounds in fp32 (relative to |x|+|c|), and the row constant is subtracted
              // from scores of its own magnitude (T64: + one rounding where the converters add the row's two halves)
              E += 1.2e-7f * (__fsqrt_ru(norms[3 * TM + r]) * cmax + p.stats->yabs * xn) +
                   (T64 ? 6.0e-7f : 4.8e-7f) * (goff + xn * cmax);
            }
            float mg = 2.f * E * 1.001f + 1e-30f;
            if (MODE == 2) mg += knn_extra;
            if (!(mg < 1.0e30f)) fl |= 1u;                                  // NaN / Inf somewhere in the row
            return mg;
          };
          if (MODE < 2) {
#pragma unroll
            for (int hh = 0; hh < 2; hh++) {
              uint32_t fl = 0;
              const float mg = row_margin(qrow + 8 * hh, fl);
              if ((lane & 3) == 0) fin[FIN_MARGIN + frow + 8 * hh] = mg;
              *fst |= fl << (8 + 8 * hh);
            }
            __syncwarp();
          } else {
            margin = row_margin(row, flags);
          }
          if (MODE == 2) {
            mmax = fmaxf(mmax, margin);
            if (p.knn_first_pass && seg == 1) {
              // threshold sweep done: both column halves of the row adopt the merged top-kk (the partner half is
              // lane ^ 2 of the same warp)
              float mg[KNN_MAX_KK];
              if constexpr (T64) {
                // the row's four parts sit in both consumer warpgroups: every part's buckets are complete before any
                // is read, and read before a warpgroup starts its next tile, which resets them
                ptx::named_bar_sync(1, N_EPI_WARPS * 32);
                knn_select_buckets4(reinterpret_cast<float*>(smem + L.list) + row + 16 * 256, p.kk, goff, mg);
                ptx::named_bar_sync(1, N_EPI_WARPS * 32);
              } else {
                __syncwarp();
                knn_select_buckets(topk + 16 * 256, reinterpret_cast<float*>(smem + L.list) + ((1 - h) * TM + row) + 16 * 256,
                                   p.kk, goff, mg);
                __syncwarp();
              }
              for (int j = 0; j < p.kk; j++) topk[j * 256] = mg[j];
              M = mg[p.kk - 1];
            }
          }
        }
        if (MODE < 2) {
          // Lloyd / Yinyang candidate epilogue on the fragment as it lands: mask bit b = 2j + e of row hh (R0 / R1) is
          // acc[j*4 + hh*2 + e], column 8j + 2t + e of the n-tile.  Any fixed column order would do: the running row
          // maximum and the "within margin" bits do not depend on it, and the emitter decodes bits into columns.
          if (it.seg_last()) si++;
#if KMB_KO == 7
          if (MODE == 0) {   // timing build: the accumulators are loaded, the ALU work on them is skipped
            uint32_t x0 = 0, x1 = 0;
#pragma unroll
            for (int j = 0; j < NACC / 4; j += 4) { x0 ^= __float_as_uint(acc[j * 4]); x1 ^= __float_as_uint(acc[j * 4 + 2]); }
            Mr[0] = fmaxf(Mr[0], __uint_as_float(x0 & 0x3fffffffu));
            Mr[1] = fmaxf(Mr[1], __uint_as_float(x1 & 0x3fffffffu));
            continue;
          }
#endif
          float cm[2], thr[2];    // this lane's chunk maximum (32 columns; T64: 16) and the row's threshold
          uint32_t mask[2];
#pragma unroll
          for (int hh = 0; hh < 2; hh++) {
            auto v = [&](int b) { return acc[(b >> 1) * 4 + hh * 2 + (b & 1)]; };
            // chunk maximum with three-input maxima: 15 instructions per 32 columns
            if constexpr (T64) {
              float u[5];
#pragma unroll
              for (int i = 0; i < 5; i++) u[i] = ptx::fmax3(v(3 * i), v(3 * i + 1), v(3 * i + 2));
              cm[hh] = fmaxf(ptx::fmax3(u[0], u[1], u[2]), ptx::fmax3(u[3], u[4], v(15)));
            } else {
              float u[10];
#pragma unroll
              for (int i = 0; i < 10; i++) u[i] = ptx::fmax3(v(3 * i), v(3 * i + 1), v(3 * i + 2));
              cm[hh] = fmaxf(ptx::fmax3(ptx::fmax3(u[0], u[1], u[2]), ptx::fmax3(u[3], u[4], u[5]), ptx::fmax3(u[6], u[7], u[8])),
                             ptx::fmax3(u[9], v(30), v(31)));
            }
            if (MODE == 0) {
              // quad all-reduce: the running maximum of the whole row (T64: of the warpgroup's columns of the row)
              float qm = fmaxf(cm[hh], __shfl_xor_sync(0xffffffffu, cm[hh], 1));
              qm = fmaxf(qm, __shfl_xor_sync(0xffffffffu, qm, 2));
              Mr[hh] = fmaxf(Mr[hh], qm);
              thr[hh] = fminf(Mr[hh], cap) - fin[FIN_MARGIN + frow + 8 * hh];
            } else {
              // (largest, second largest) of the quad's four chunk maxima, merged into the row's running pair.  The
              // chunks of the four lanes and of different n-tiles are disjoint column sets, so two distinct columns
              // reach the second value of the pair: M2 is a lower bound of the row's second best score.  (Merged
              // over the quad rather than kept per lane: the lane's own pair is valid too, but looser.)
              const float o = __shfl_xor_sync(0xffffffffu, cm[hh], 1);
              const float a1 = fmaxf(cm[hh], o), a2 = fminf(cm[hh], o);
              const float b1 = __shfl_xor_sync(0xffffffffu, a1, 2), b2 = __shfl_xor_sync(0xffffffffu, a2, 2);
              const float q1 = fmaxf(a1, b1), q2 = fmaxf(fminf(a1, b1), fmaxf(a2, b2));
              M2r[hh] = ptx::fmax3(M2r[hh], q2, fminf(Mr[hh], q1));
              Mr[hh] = fmaxf(Mr[hh], q1);
              thr[hh] = fminf(M2r[hh], cap) - fin[FIN_MARGIN + frow + 8 * hh];
            }
            // candidate mask: d = v - thr as packed pairs, then the sign bits are shifted in with one funnel shift per
            // column; bit (31 - b) of (c0 << 16 | c1) = sign of d_b = "bit b is below the threshold".  NaN scores only
            // occur in rows whose margin is not finite (flag 1).
            const uint64_t nthr2 = ptx::pack2(-thr[hh], -thr[hh]);
            uint32_t c0 = 0, c1 = 0;   // two 16-column chains (shorter dependency chains; T64: two 8-column chains)
#pragma unroll
            for (int j = 0; j < NACC / 4; j++) {
              float x, y;
              ptx::unpack2(ptx::fadd2(ptx::pack2(v(2 * j), v(2 * j + 1)), nthr2), x, y);
              if (j < NACC / 8) {
                c0 = __funnelshift_l(__float_as_uint(x), c0, 1);
                c0 = __funnelshift_l(__float_as_uint(y), c0, 1);
              } else {
                c1 = __funnelshift_l(__float_as_uint(x), c1, 1);
                c1 = __funnelshift_l(__float_as_uint(y), c1, 1);
              }
            }
            // T64: bit (15 - b) of (c0 << 8 | c1) is the sign of d_b; shifted to the top so the reversal leaves 16 bits
            if constexpr (T64) mask[hh] = __brev(~((c0 << 8) | c1) << 16);
            else mask[hh] = __brev(~((c0 << 16) | c1));
          }
          // one entry per n-tile in which either row holds a candidate in this lane's columns
          if (mask[0] | mask[1]) {
            constexpr uint32_t A = LIST_ARRAY / 4;
            uint32_t st = *fst, c = st & 0xffu;
            if (c >= LIST_LEN - 1) c = compact_list(lst, lnt, c, thr[0], thr[1]);   // rare: drop entries below the risen thresholds
            if (c < LIST_LEN) {
              lst[c * 256] = __float_as_uint(cm[0]);
              lst[A + c * 256] = __float_as_uint(cm[1]);
              lst[2 * A + c * 256] = mask[0];
              lst[3 * A + c * 256] = mask[1];
              lnt[c * 256] = static_cast<uint16_t>(n);
              c++;
            } else {
              st |= (mask[0] ? 2u << 8 : 0u) | (mask[1] ? 2u << 16 : 0u);   // the row's candidate set is incomplete
            }
            *fst = (st & ~0xffu) | c;
          }
          continue;
        }
        if constexpr (MODE == 2 && T64) {
          // 64-row tiles: this thread gets the 32 columns of its part (regroup_quad_t64) and runs the steps of the
          // 128-row epilogue below on that one chunk; threshold buckets (n-tile % 4, 4-column group), 32 per part
          uint32_t r[32];
#if KMB_KO != 1
          regroup_quad_t64(acc, lane, r);
#else
          for (int jj = 0; jj < 32; jj++) r[jj] = __float_as_uint(-64.f * static_cast<float>(n * 128 + kpart * 32 + jj + 1));
#endif
          float t0[8];
#pragma unroll
          for (int i = 0; i < 8; i++)
            t0[i] = fmaxf(fmaxf(__uint_as_float(r[4 * i]), __uint_as_float(r[4 * i + 1])),
                          fmaxf(__uint_as_float(r[4 * i + 2]), __uint_as_float(r[4 * i + 3])));
          const float cm0 = fmaxf(fmaxf(fmaxf(t0[0], t0[1]), fmaxf(t0[2], t0[3])), fmaxf(fmaxf(t0[4], t0[5]), fmaxf(t0[6], t0[7])));
          if (p.knn_first_pass && seg == 0) {
            float* bk = topk + (16 + 8 * (n & 3)) * 256;
#pragma unroll
            for (int i = 0; i < 8; i++) bk[i * 256] = fmaxf(bk[i * 256], t0[i]);
          } else if (!p.knn_first_pass && cm0 > M + goff) {
#pragma unroll
            for (int i = 0; i < 8; i++)
              if (t0[i] - goff > M) M = knn_topk_insert(topk, p.kk, t0[i] - goff);
          }
          const float thr = (M - margin) + goff;
          const uint64_t nthr2 = ptx::pack2(-thr, -thr);
          uint32_t c00 = 0, c01 = 0;
#pragma unroll
          for (int jj = 0; jj < 32; jj += 2) {
            float x0, y0;
            ptx::unpack2(ptx::fadd2(ptx::pack2(__uint_as_float(r[jj]), __uint_as_float(r[jj + 1])), nthr2), x0, y0);
            if (jj < 16) {
              c00 = __funnelshift_l(__float_as_uint(x0), c00, 1);
              c00 = __funnelshift_l(__float_as_uint(y0), c00, 1);
            } else {
              c01 = __funnelshift_l(__float_as_uint(x0), c01, 1);
              c01 = __funnelshift_l(__float_as_uint(y0), c01, 1);
            }
          }
          const uint32_t mask0 = __brev(~((c00 << 16) | c01));
          // chunk id n * 4 + part: the column decode of expand_kernel (128 n + 64 (part >> 1) + 32 (part & 1)) holds
          if (klive && !(p.knn_first_pass && seg == 0) && mask0)
            cnt = knn_append(kent, cnt, M, cm0 - goff, mask0, static_cast<uint32_t>(n) * 4 + kpart, margin, &flags);
          if (it.seg_last()) { si++; seg++; }
          continue;
        }
        if constexpr (MODE == 3 && T64) {
          // 64-row tiles: this thread's part 2g + h of the row is 32 consecutive columns (regroup_quad_t64), the table
          // quads 8 (2g + h) .. +7 of the n-tile.  The lanes of one warp hold two different quarters (h = (l % 4) / 2),
          // so every lane folds its own 8 quads along its own group ids; the runs of a group split at part boundaries
          // and each piece flushes its own bound (yy_fold_groups)
          uint32_t r[32];
#if KMB_KO != 1
          regroup_quad_t64(acc, lane, r);
#else
          for (int jj = 0; jj < 32; jj++) r[jj] = __float_as_uint(-64.f * static_cast<float>(n * 128 + kpart * 32 + jj + 1));
#endif
          float qm[8];
#pragma unroll
          for (int i = 0; i < 8; i++)
            qm[i] = fmaxf(ptx::fmax3(__uint_as_float(r[4 * i]), __uint_as_float(r[4 * i + 1]), __uint_as_float(r[4 * i + 2])),
                          __uint_as_float(r[4 * i + 3]));
          uint32_t gq[8];
          {
            const uint4* src = reinterpret_cast<const uint4*>(p.yy_qgroup) + static_cast<size_t>(n) * 8 + kpart * 2;
            const uint4 v0 = __ldg(src), v1 = __ldg(src + 1);
            gq[0] = v0.x; gq[1] = v0.y; gq[2] = v0.z; gq[3] = v0.w;
            gq[4] = v1.x; gq[5] = v1.y; gq[6] = v1.z; gq[7] = v1.w;
          }
          yy_fold_groups<8>(p, qm, gq, ylive && !(flags & 1u), gown, 0.5f * margin /* >= E */, xa2lo, yb);
          if (it.seg_last()) si++;
          continue;
        }
        // MODE 2 / 3: this thread gets columns h*64 .. h*64+63 of its row (quad shuffles, see regroup_quad)
        uint32_t r0[32], r1[32];
#if KMB_KO != 1
        if constexpr (MODE >= 2 && !T64) regroup_quad(acc, lane, r0, r1);   // (MODE 0 / 1 never reach this point)
#else
        for (int jj = 0; jj < 32; jj++) {   // stand-in values: strictly decreasing, 64 apart -> one candidate per row
          r0[jj] = __float_as_uint(-64.f * static_cast<float>(n * 128 + h * 64 + jj + 1));
          r1[jj] = __float_as_uint(-64.f * static_cast<float>(n * 128 + h * 64 + 32 + jj + 1));
        }
#endif
        if (MODE == 3) {
          // quad maxima (2 instructions per 4 columns), folded into per-group maxima along the (warp-uniform) group ids
          // of this 64-column half; every finished group turns into a lower bound of the distance
          float qm[16];
#pragma unroll
          for (int i = 0; i < 8; i++) {
            qm[i] = fmaxf(ptx::fmax3(__uint_as_float(r0[4 * i]), __uint_as_float(r0[4 * i + 1]), __uint_as_float(r0[4 * i + 2])),
                          __uint_as_float(r0[4 * i + 3]));
            qm[8 + i] = fmaxf(ptx::fmax3(__uint_as_float(r1[4 * i]), __uint_as_float(r1[4 * i + 1]), __uint_as_float(r1[4 * i + 2])),
                              __uint_as_float(r1[4 * i + 3]));
          }
          uint32_t gq[16];
          {
            const uint4* src = reinterpret_cast<const uint4*>(p.yy_qgroup) + (static_cast<size_t>(n) * 2 + h) * 4;
#pragma unroll
            for (int i = 0; i < 4; i++) {
              const uint4 v = __ldg(src + i);
              gq[4 * i] = v.x; gq[4 * i + 1] = v.y; gq[4 * i + 2] = v.z; gq[4 * i + 3] = v.w;
            }
          }
          // (the group ids are the same in every lane of one column half: the table layout is the same for every row)
          yy_fold_groups<16>(p, qm, gq, ylive && !(flags & 1u), gown, 0.5f * margin /* >= E */, xa2lo, yb);
          if (it.seg_last()) si++;
          continue;
        }
        if (MODE == 2) {
          // MODE 2: maxima of the 4-column groups and of the two 32-column chunks
          float t0[8], t1[8];
#pragma unroll
          for (int i = 0; i < 8; i++) {
            t0[i] = fmaxf(fmaxf(__uint_as_float(r0[4 * i]), __uint_as_float(r0[4 * i + 1])),
                          fmaxf(__uint_as_float(r0[4 * i + 2]), __uint_as_float(r0[4 * i + 3])));
            t1[i] = fmaxf(fmaxf(__uint_as_float(r1[4 * i]), __uint_as_float(r1[4 * i + 1])),
                          fmaxf(__uint_as_float(r1[4 * i + 2]), __uint_as_float(r1[4 * i + 3])));
          }
          const float cm0 = fmaxf(fmaxf(fmaxf(t0[0], t0[1]), fmaxf(t0[2], t0[3])), fmaxf(fmaxf(t0[4], t0[5]), fmaxf(t0[6], t0[7])));
          const float cm1 = fmaxf(fmaxf(fmaxf(t1[0], t1[1]), fmaxf(t1[2], t1[3])), fmaxf(fmaxf(t1[4], t1[5]), fmaxf(t1[6], t1[7])));
          // kk distinct columns reach the kk-th largest 4-column-group maximum (first level of the max tree): a
          // lower bound of the kk-th best score; finer than whole chunks because near neighbours sit close together
          // in the table.  M and the list live in g-space (score - goff).
          if (p.knn_first_pass && seg == 0) {
            // threshold sweep: bucket (block parity, 4-column group) <- max; raw scores, the row constant is
            // subtracted once at the end of the sweep
            float* bk = topk + (16 + 16 * (n & 1)) * 256;
#pragma unroll
            for (int i = 0; i < 8; i++) {
              bk[i * 256] = fmaxf(bk[i * 256], t0[i]);
              bk[(8 + i) * 256] = fmaxf(bk[(8 + i) * 256], t1[i]);
            }
          } else if (!p.knn_first_pass) {
            const float lim = M + goff;
            if (cm0 > lim) {
#pragma unroll
              for (int i = 0; i < 8; i++)
                if (t0[i] - goff > M) M = knn_topk_insert(topk, p.kk, t0[i] - goff);
            }
            if (cm1 > lim) {
#pragma unroll
              for (int i = 0; i < 8; i++)
                if (t1[i] - goff > M) M = knn_topk_insert(topk, p.kk, t1[i] - goff);
            }
          }
          const float thr = (M - margin) + goff;
          // candidate masks: d_j = v_j - thr as packed pairs, then the sign bits are shifted into a mask with one funnel
          // shift per column
          uint32_t nc0, nc1;
          {
            const uint64_t nthr2 = ptx::pack2(-thr, -thr);
            uint32_t c00 = 0, c01 = 0, c10 = 0, c11 = 0;   // two 16-column chains per chunk (shorter dependency chains)
#pragma unroll
            for (int jj = 0; jj < 32; jj += 2) {
              float x0, y0, x1, y1;
              ptx::unpack2(ptx::fadd2(ptx::pack2(__uint_as_float(r0[jj]), __uint_as_float(r0[jj + 1])), nthr2), x0, y0);
              ptx::unpack2(ptx::fadd2(ptx::pack2(__uint_as_float(r1[jj]), __uint_as_float(r1[jj + 1])), nthr2), x1, y1);
              if (jj < 16) {
                c00 = __funnelshift_l(__float_as_uint(x0), c00, 1);
                c00 = __funnelshift_l(__float_as_uint(y0), c00, 1);
                c10 = __funnelshift_l(__float_as_uint(x1), c10, 1);
                c10 = __funnelshift_l(__float_as_uint(y1), c10, 1);
              } else {
                c01 = __funnelshift_l(__float_as_uint(x0), c01, 1);
                c01 = __funnelshift_l(__float_as_uint(y0), c01, 1);
                c11 = __funnelshift_l(__float_as_uint(x1), c11, 1);
                c11 = __funnelshift_l(__float_as_uint(y1), c11, 1);
              }
            }
            // bit (31 - j) of (c?0 << 16 | c?1) = sign of d_j = "column j is below the threshold"
            nc0 = (c00 << 16) | c01;
            nc1 = (c10 << 16) | c11;
          }
          const uint32_t mask0 = __brev(~nc0), mask1 = __brev(~nc1);
          if (klive && !(p.knn_first_pass && seg == 0)) {
            if (mask0)
              cnt = knn_append(kent, cnt, M, cm0 - goff, mask0, static_cast<uint32_t>(n) * 4 + h * 2, margin, &flags);
            if (mask1)
              cnt = knn_append(kent, cnt, M, cm1 - goff, mask1, static_cast<uint32_t>(n) * 4 + h * 2 + 1, margin, &flags);
          }
          if (it.seg_last()) { si++; seg++; }
        }
      }
      if (MODE == 2) {
        if (klive) {
          for (int j = 0; j < p.kk; j++) p.knn_topk[static_cast<size_t>(j) * p.knn_stride + kslot] = topk[j * 256];
          p.knn_cnt[kslot] = cnt;
          p.knn_flags[kslot] = flags;
          // exact distance to the kk-th nearest candidate seen so far, upper bound in the caller's units:
          // every recorded score is within its margin of g = -s^2 d^2 / 2
          const float sc = p.stats->scale;
          const float d2 = fmaxf(0.f, -2.f * (M - mmax));
          p.knn_dub[kslot] = (M > -INFINITY && !flags) ? __fsqrt_ru(d2) / sc * 1.0001f : INFINITY;
        }
        ti++;
        continue;
      }
      if (MODE == 3) {
        // rows the filter cannot bound (non-finite data, scores beyond the sentinel range): exact refresh of the row, listed
        // once, by its part 0 (the flag comes from the row's norms, the same in every part)
        if (ylive && (flags & 1u) && kpart == 0)
          p.ovf_rows[atomicAdd(&p.counters[CNT_OVF], 1u)] = static_cast<uint32_t>(tile * TR + row);
        ti++;
        continue;
      }
      // publish the per-row maxima (the same in the four lanes of a quad); the emitter warps merge the four lists of
      // a row and write the results
      if ((lane & 3) == 0) {
#pragma unroll
        for (int hh = 0; hh < 2; hh++) {
          fin[FIN_M + frow + 8 * hh] = Mr[hh];
          if (MODE == 1) fin[FIN_M2 + frow + 8 * hh] = M2r[hh];   // T64: one pair per (row, warpgroup)
        }
      }
      __syncwarp();
      if (lane == 0) ptx::mbar_arrive(&bars[BAR_EMIT_FULL + par]);
      ti++;
    }
  }
  // no warp leaves while TMA copies into this CTA's shared memory may still be in flight
  __syncthreads();
}

template <int NKB, int MODE>
__global__ void __launch_bounds__(N_THREADS, 1)
tc_assign_kernel(const __grid_constant__ CUtensorMap tmap_b, const Params p) {
  tc_assign_body<NKB, MODE, false>(tmap_b, p);
}

// the mini-batch pass over a row list (ROWS above): MODE 0 with the samples read through p.rows
template <int NKB>
__global__ void __launch_bounds__(N_THREADS, 1)
tc_assign_rows_kernel(const __grid_constant__ CUtensorMap tmap_b, const Params p) {
  tc_assign_body<NKB, 0, true>(tmap_b, p);
}

}  // namespace tc

// ---------------------------------------------------------------------------------------------------
// exact re-check of (row, candidate) pairs + per-row reduction
// ---------------------------------------------------------------------------------------------------
template <int METRIC, int MODE>   // MODE 0: Lloyd ranking score; MODE 1: true distance (Yinyang bounds)
__global__ void __launch_bounds__(128)
recheck_pairs_kernel(const float* __restrict__ X, const float* __restrict__ C,
                     const float* __restrict__ csq, int D, const uint32_t* __restrict__ pair_row,
                     const uint32_t* __restrict__ pair_cand, const uint32_t* __restrict__ d_npairs,
                     uint32_t max_pairs, uint32_t n, uint32_t K, float* __restrict__ pair_score) {
  // 128 (row, candidate) pairs per CTA; features stream through shared memory 32 at a time.
  // Staging: every thread issues 16 independent 16-byte loads per chunk (8 lanes cover one 128-byte row segment).  The
  // loads of chunk i+1 are issued BEFORE the sequential Kahan loop of chunk i (32 features x a 4-instruction dependent
  // chain per pair), so the global-memory latency of a chunk hides behind the previous chunk's arithmetic (round 2:
  // load -> store -> compute ran back to back, 233 us for 0.92 M pairs at the headline shape).
  __shared__ float sX[32 * 129];     // [feature][pair]   (+1 padding: conflict-free both ways)
  __shared__ float sC[128 * 33];     // [pair][feature]
  __shared__ uint32_t s_row[128], s_cand[128];
  const uint32_t np = min(*d_npairs, max_pairs);
  const int nchunks = (D + 31) / 32;
  for (uint32_t tile0 = blockIdx.x * 128; tile0 < np; tile0 += gridDim.x * 128) {
    const uint32_t pidx = tile0 + threadIdx.x;
    const bool active = pidx < np;
    __syncthreads();
    // (slots past the last complete row group may hold stale data: stay in bounds)
    s_row[threadIdx.x] = active ? min(pair_row[pidx], n - 1) : 0;
    s_cand[threadIdx.x] = active ? min(pair_cand[pidx], K - 1) : 0;
    __syncthreads();
    // the whole sample row of this thread's pair is requested from DRAM now, line after line (one open DRAM page per
    // row), so that the chunk loads below -- 128 bytes of the row per chunk, spread over the chunk loop -- hit L2
    // instead of making eight scattered DRAM accesses per row
    if (active) {
      const char* xr = reinterpret_cast<const char*>(X + static_cast<size_t>(s_row[threadIdx.x]) * D);
      for (int b = 128; b < D * 4; b += 128) asm volatile("prefetch.global.L2 [%0];" ::"l"(xr + b));
    }
    Kahan k;
    float4 v[16];
    auto load_chunk = [&](int f0) {
      const int fl = min(32, D - f0);
#pragma unroll
      for (int i = 0; i < 16; i++) {
        const int idx = i * 128 + threadIdx.x;  // [which(1)][pair(7)][quad(3)]
        const int q = idx & 7, e = (idx >> 3) & 127, which = idx >> 10;
        const float* src = which ? C + static_cast<size_t>(s_cand[e]) * D : X + static_cast<size_t>(s_row[e]) * D;
        v[i] = (q * 4 < fl) ? *reinterpret_cast<const float4*>(src + f0 + q * 4) : make_float4(0.f, 0.f, 0.f, 0.f);
      }
    };
    load_chunk(0);
    for (int ch = 0; ch < nchunks; ch++) {
      const int fl = min(32, D - ch * 32);
      __syncthreads();                      // the previous chunk has been consumed
#pragma unroll
      for (int i = 0; i < 16; i++) {
        const int idx = i * 128 + threadIdx.x;
        const int q = idx & 7, e = (idx >> 3) & 127, which = idx >> 10;
        if (which) {
          float* d = sC + e * 33 + q * 4;
          d[0] = v[i].x; d[1] = v[i].y; d[2] = v[i].z; d[3] = v[i].w;
        } else {
          float* d = sX + (q * 4) * 129 + e;
          d[0] = v[i].x; d[129] = v[i].y; d[258] = v[i].z; d[387] = v[i].w;
        }
      }
      __syncthreads();
      if (ch + 1 < nchunks) load_chunk((ch + 1) * 32);   // in flight during the loop below
      if (active)
        for (int f = 0; f < fl; f++) {
          if (MODE == 1 && METRIC == 0) k.sqdiff(sX[f * 129 + threadIdx.x], sC[threadIdx.x * 33 + f]);
          else k.mac(sX[f * 129 + threadIdx.x], sC[threadIdx.x * 33 + f]);
        }
    }
    if (active)
      pair_score[pidx] = MODE == 1 ? finalize_distance<METRIC>(k.sum)
                                   : lloyd_score<METRIC>(k.sum, csq[s_cand[threadIdx.x]]);
  }
}

__global__ void recheck_reduce_kernel(const uint32_t* __restrict__ rowq, const uint32_t* __restrict__ d_nrowq,
                                      const uint32_t* __restrict__ pair_cand,
                                      const float* __restrict__ pair_score, uint32_t* __restrict__ result,
                                      uint32_t* __restrict__ assign, uint32_t* __restrict__ prev,
                                      uint32_t* __restrict__ d_changed) {
  const uint32_t nq = *d_nrowq;
  uint32_t nchanged = 0;
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < nq; i += gridDim.x * blockDim.x) {
    const uint32_t row = rowq[3 * i], base = rowq[3 * i + 1], cnt = rowq[3 * i + 2];
    if (cnt == 0) continue;  // neutralised slot (pair queue was full; the row is on the overflow list)
    float best = FLT_MAX;
    uint32_t arg = UINT32_MAX;
    for (uint32_t j = 0; j < cnt; j++) {
      const float sc = pair_score[base + j];
      const uint32_t c = pair_cand[base + j];
      // strict '<' in ascending centroid order == lowest index among equal scores
      if (sc < best || (sc == best && c < arg)) {
        best = sc;
        arg = c;
      }
    }
    if (assign) {
      if (arg != UINT32_MAX) nchanged += tc::commit_assignment(assign, prev, row, arg);
    } else {
      result[row] = (arg == UINT32_MAX) ? kUntouched : arg;
    }
  }
  if (assign) {
    nchanged = __reduce_add_sync(0xffffffffu, nchanged);
    if ((threadIdx.x & 31) == 0 && nchanged) atomicAdd(d_changed, nchanged);
  }
}

// bookkeeping for the rows that took the full exact pass (their winners are in result[])
__global__ void finalize_rows_kernel(const uint32_t* __restrict__ rows, const uint32_t* __restrict__ d_nrows,
                                     const uint32_t* __restrict__ result, uint32_t* __restrict__ assign,
                                     uint32_t* __restrict__ prev, uint32_t* __restrict__ d_changed) {
  const uint32_t nr = *d_nrows;
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < nr; i += gridDim.x * blockDim.x) {
    const uint32_t row = rows[i], r = result[row];
    if (r != kUntouched && tc::commit_assignment(assign, prev, row, r)) atomicAdd(d_changed, 1u);
  }
}

// ---------------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------------
struct TcPlan {
  int metric, D, device, nkb, nt;
  uint32_t K, max_n, max_pairs;
  __half* table = nullptr;
  __half* aug_blob = nullptr;
  tc::Stats* stats = nullptr;
  float* cnorm2 = nullptr;         // cosine: ||c||^2 (the reference's 'csqr' is the constant 1 there); L2: ||c - mu||^2
  double* musum = nullptr;         // [D] column sums of the valid centroids, followed by the valid-row count
  float* neg_mu_s = nullptr;       // [nkb*64] centring term (L2), see Params::neg_mu_s
  bool inject_error = false;       // test hook (KMCUDA_B200_INJECT_PIPELINE_ERROR=1): report a timed-out barrier
  // Yinyang bounds refresh (MODE 3): group-sorted table layout, built once per run by tc_yy_layout()
  int nt3 = 0;
  uint32_t G3 = 0;
  __half* table3 = nullptr;
  __half* aug_blob3 = nullptr;
  uint32_t* yy_perm = nullptr;     // [nt3*128] table row -> centroid (UINT32_MAX = padding)
  uint32_t* yy_qgroup = nullptr;   // [nt3*32] group of every 4-column quad
  uint32_t* yy_goff = nullptr;     // [G+1] CSR of the group members
  uint32_t* yy_gmem = nullptr;     // [K]
  uint32_t yy_max_gsize = 0;       // members of the largest group
  CUtensorMap tmap3;
  uint32_t *pair_row = nullptr, *pair_cand = nullptr, *rowq = nullptr, *ovf_rows = nullptr, *counters = nullptr;
  float* pair_score = nullptr;
  uint32_t* h_counters = nullptr;  // pinned
  unsigned* prep_barrier = nullptr;   // {arrivals, generation} of tc_prep_fused_kernel's grid barrier (zero between launches)
  CUtensorMap tmap;     // fp16 centroid table
  int num_sms = 132;
  size_t smem_bytes = 0;
  // CUDA-event pairs around the main kernel of the most recent passes (bench.py roofline)
  static constexpr int kEvRing = 64;
  cudaEvent_t ev0[kEvRing] = {}, ev1[kEvRing] = {};
  uint64_t passes = 0;
  bool capturing = false;          // the pass is being captured into a CUDA graph (Shard::assign): events are recorded as
  int graph_slot = -1;             // external event nodes into one fixed slot, which every replay of the graph refreshes
};

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*,
                                  CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion,
                                  CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode_fn() {
  static EncodeTiledFn fn = nullptr;
  if (!fn) {
    void* ptr = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &ptr, cudaEnableDefault, &qres) == cudaSuccess &&
        qres == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(ptr);
  }
  return fn;
}

// fp16 table [rows][nkb*64] as the B operand: boxes of 64 features x 128 rows, 128-byte swizzle
static cudaError_t encode_table_map(CUtensorMap* map, const __half* table, size_t rows, int nkb) {
  using namespace tc;
  EncodeTiledFn enc = get_encode_fn();
  if (!enc) return cudaErrorNotSupported;
  cuuint64_t gdim[2] = {static_cast<cuuint64_t>(nkb * KB), static_cast<cuuint64_t>(rows)};
  cuuint64_t gstride[1] = {static_cast<cuuint64_t>(nkb * KB) * sizeof(__half)};
  cuuint32_t box[2] = {KB, TN};
  cuuint32_t estr[2] = {1, 1};
  CUresult cr = enc(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, const_cast<__half*>(table), gdim, gstride, box, estr,
                    CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                    CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return cr == CUDA_SUCCESS ? cudaSuccess : cudaErrorInvalidValue;
}

// The main kernels, tc_kernels[nkb - 1][MODE]: tc_assign_kernel<nkb, MODE> for MODE 0..3, then at [4] the row list
// (tc_assign_rows_kernel<nkb>, MODE 0), for nkb 1..16
typedef void (*TcKernel)(CUtensorMap, tc::Params);
typedef std::array<TcKernel, 5> TcKernels;
template <class F, int... I>
static std::array<TcKernels, sizeof...(I)> table_over_nkb(F row, std::integer_sequence<int, I...>) {
  return {row(std::integral_constant<int, I + 1>{})...};
}
static const auto tc_kernels = table_over_nkb([](auto nkb) {
  return TcKernels{tc::tc_assign_kernel<decltype(nkb)::value, 0>, tc::tc_assign_kernel<decltype(nkb)::value, 1>,
                   tc::tc_assign_kernel<decltype(nkb)::value, 2>, tc::tc_assign_kernel<decltype(nkb)::value, 3>,
                   tc::tc_assign_rows_kernel<decltype(nkb)::value>};
}, std::make_integer_sequence<int, tc::MAX_TILE64_NKB>{});

// nkb lies in 1..16 for every plan (tc_supported) and k-NN call (tc_knn_supported)
static void tc_launch(int mode, bool rows, int nkb, unsigned grid, size_t smem, cudaStream_t st, const CUtensorMap& tb,
                      const tc::Params& prm) {
  tc_kernels[nkb - 1][rows ? 4 : mode]<<<grid, tc::N_THREADS, smem, st>>>(tb, prm);
}
// every kernel a plan of this nkb may launch (MODE 0..3 and the row list) may use `bytes` of dynamic shared memory
static cudaError_t tc_set_smem_attr(int bytes, int nkb) {
  if (nkb < 1 || nkb > tc::MAX_TILE64_NKB) return cudaErrorInvalidValue;
  for (int k = 0; k < 5; k++) {
    const cudaError_t e =
        cudaFuncSetAttribute(tc_kernels[nkb - 1][k], cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
    if (e != cudaSuccess) return e;
  }
  return cudaSuccess;
}

// exact re-check of the queued (row, candidate) pairs in the metric of the run: MODE 0 Lloyd ranking score, MODE 1 true
// distance (see recheck_pairs_kernel)
template <int MODE>
static void launch_recheck_pairs(int metric, unsigned grid, cudaStream_t st, const float* X, const float* C,
                                 const float* csq, int D, const uint32_t* pair_row, const uint32_t* pair_cand,
                                 const uint32_t* d_npairs, uint32_t max_pairs, uint32_t n, uint32_t K,
                                 float* pair_score) {
  (metric == 1 ? recheck_pairs_kernel<1, MODE> : recheck_pairs_kernel<0, MODE>)<<<grid, 128, 0, st>>>(
      X, C, csq, D, pair_row, pair_cand, d_npairs, max_pairs, n, K, pair_score);
}

// (the pinned allocation below is milliseconds: a plan is created by every kmeans_cuda call, so freed blocks are
// kept per process)
static std::mutex g_pinned_mu;
static std::vector<uint32_t*> g_pinned_free;   // CNT_N-word pinned blocks of destroyed plans
static uint32_t* pinned_counters_alloc() {
  {
    std::lock_guard<std::mutex> lk(g_pinned_mu);
    if (!g_pinned_free.empty()) {
      uint32_t* p = g_pinned_free.back();
      g_pinned_free.pop_back();
      return p;
    }
  }
  void* p = nullptr;
  if (cudaHostAlloc(&p, sizeof(uint32_t) * tc::CNT_N, cudaHostAllocPortable) != cudaSuccess) {
    cudaGetLastError();
    return nullptr;
  }
  return static_cast<uint32_t*>(p);
}
static void pinned_counters_free(uint32_t* p) {
  if (!p) return;
  std::lock_guard<std::mutex> lk(g_pinned_mu);
  g_pinned_free.push_back(p);
}

// every mode up to D = 1024 (512 < D <= 1024 on 64-row tiles; k-NN keeps its own checks in tc_knn_supported)
bool tc_supported(int metric, uint32_t n, int D, uint32_t K) {
  if (D < 4 || D % 4 != 0 || D > tc::MAX_TILE64_NKB * tc::KB) return false;   // TMA row pitch must be 16-byte aligned
  if (K < 2 || K > 16383u * 128u) return false;        // chunk ids are 16 bit (4 per n-tile)
  if (n == 0) return false;
  return true;
}

void tc_plan_destroy(TcPlan* p) {
  if (!p) return;
  pool_free(p->table);
  pool_free(p->aug_blob);
  pool_free(p->stats);
  pool_free(p->cnorm2);
  pool_free(p->musum);
  pool_free(p->neg_mu_s);
  pool_free(p->table3);
  pool_free(p->aug_blob3);
  pool_free(p->yy_perm);
  pool_free(p->yy_qgroup);
  pool_free(p->yy_goff);
  pool_free(p->yy_gmem);
  pool_free(p->pair_row);
  pool_free(p->pair_cand);
  pool_free(p->pair_score);
  pool_free(p->rowq);
  pool_free(p->ovf_rows);
  pool_free(p->counters);
  pool_free(p->prep_barrier);
  pinned_counters_free(p->h_counters);
  for (int i = 0; i < TcPlan::kEvRing; i++) {
    if (p->ev0[i]) cudaEventDestroy(p->ev0[i]);
    if (p->ev1[i]) cudaEventDestroy(p->ev1[i]);
  }
  delete p;
}

cudaError_t tc_plan_create(TcPlan** out, int metric, uint32_t max_n, int D, uint32_t K, int device) {
  using namespace tc;
  TcPlan* p = new TcPlan;
  p->metric = metric;
  p->D = D;
  p->K = K;
  p->device = device;
  p->max_n = max_n;
  p->nkb = (D + KB - 1) / KB;
  p->nt = static_cast<int>((K + TN - 1) / TN);
  p->max_pairs = max_n < (1u << 28) ? 10 * max_n + 1024 : 0xFFFFFFF0u;   // Lloyd needs ~0.4 n, the Yinyang top-2 mode up to ~7 n
  cudaError_t e;
#define TC_TRY(x) do { e = (x); if (e != cudaSuccess) { tc_plan_destroy(p); return e; } } while (0)
  TC_TRY(cudaDeviceGetAttribute(&p->num_sms, cudaDevAttrMultiProcessorCount, device));
  const size_t rows_pad = static_cast<size_t>(p->nt) * TN;
  TC_TRY(pool_alloc(reinterpret_cast<void**>(&p->table), rows_pad * p->nkb * KB * sizeof(__half)));
  TC_TRY(pool_alloc(reinterpret_cast<void**>(&p->aug_blob), static_cast<size_t>(p->nt) * AUG_B_BYTES));
  TC_TRY(pool_alloc(reinterpret_cast<void**>(&p->stats), sizeof(Stats)));
  TC_TRY(pool_alloc(reinterpret_cast<void**>(&p->cnorm2), sizeof(float) * K));
  TC_TRY(pool_alloc(reinterpret_cast<void**>(&p->musum), sizeof(double) * (D + 1)));
  TC_TRY(pool_alloc(reinterpret_cast<void**>(&p->neg_mu_s), sizeof(float) * mu_features(p->nkb)));
  {
    const char* ie = getenv("KMCUDA_B200_INJECT_PIPELINE_ERROR");
    p->inject_error = ie && ie[0] == '1';
  }
  TC_TRY(pool_alloc(reinterpret_cast<void**>(&p->pair_row), sizeof(uint32_t) * p->max_pairs));
  TC_TRY(pool_alloc(reinterpret_cast<void**>(&p->pair_cand), sizeof(uint32_t) * p->max_pairs));
  TC_TRY(pool_alloc(reinterpret_cast<void**>(&p->pair_score), sizeof(float) * p->max_pairs));
  TC_TRY(pool_alloc(reinterpret_cast<void**>(&p->rowq), sizeof(uint32_t) * 3 * static_cast<size_t>(max_n)));
  TC_TRY(pool_alloc(reinterpret_cast<void**>(&p->ovf_rows), sizeof(uint32_t) * static_cast<size_t>(max_n)));
  TC_TRY(pool_alloc(reinterpret_cast<void**>(&p->counters), sizeof(uint32_t) * CNT_N));
  TC_TRY(pool_alloc(reinterpret_cast<void**>(&p->prep_barrier), sizeof(unsigned) * 2));
  TC_TRY(cudaMemset(p->prep_barrier, 0, sizeof(unsigned) * 2));
  TC_TRY(cudaStreamSynchronize(nullptr));   // the passes run on non-blocking streams, which do not order against this memset
  p->h_counters = pinned_counters_alloc();
  if (!p->h_counters) { tc_plan_destroy(p); return cudaErrorMemoryAllocation; }
  memset(p->h_counters, 0, sizeof(uint32_t) * CNT_N);
  TC_TRY(encode_table_map(&p->tmap, p->table, rows_pad, p->nkb));
  for (int i = 0; i < TcPlan::kEvRing; i++) {
    TC_TRY(cudaEventCreate(&p->ev0[i]));
    TC_TRY(cudaEventCreate(&p->ev1[i]));
  }
  p->smem_bytes = smem_layout(p->nkb).total + 1024;
  TC_TRY(tc_set_smem_attr(static_cast<int>(p->smem_bytes), p->nkb));
#undef TC_TRY
  *out = p;
  return cudaSuccess;
}

// counters reset + centroid preparation (scale, fp16 table, bias blobs) + the parameter block shared by both modes
static cudaError_t tc_prepare(TcPlan* p, const float* C, const float* csq, uint32_t n, tc::Params* out,
                              cudaStream_t st, bool yy_layout = false, bool compute_csq = false) {
  using namespace tc;
  PrepArgs a;
  a.metric = p->metric;
  a.D = p->D;
  a.nkb = p->nkb;
  a.by_source = yy_layout ? 1 : 0;
  a.K = p->K;
  a.rows_pad = static_cast<uint32_t>(yy_layout ? p->nt3 : p->nt) * TN;
  a.C = C;
  a.csq = const_cast<float*>(csq);
  a.compute_csq = compute_csq ? 1 : 0;
  a.cnorm2 = p->cnorm2;
  a.musum = p->musum;
  a.neg_mu_s = p->neg_mu_s;
  a.stats = p->stats;
  a.counters = p->counters;
  a.table = yy_layout ? p->table3 : p->table;
  a.aug_blob = yy_layout ? p->aug_blob3 : p->aug_blob;
  a.gather = yy_layout ? p->yy_perm : nullptr;
  a.barrier = p->prep_barrier;
  // one table row per warp up to the number of SMs (every CTA must be resident for the grid barrier)
  const unsigned grid = std::min<unsigned>(static_cast<unsigned>(p->num_sms), std::max(1u, (a.rows_pad + 7u) / 8u));
  tc_prep_fused_kernel<<<grid, 256, 0, st>>>(a);
  Params prm;
  prm.n = n;
  prm.D = p->D;
  prm.K = p->K;
  prm.nkb = p->nkb;
  prm.nt = yy_layout ? p->nt3 : p->nt;
  prm.ntiles = (n + tile_rows(p->nkb) - 1) / tile_rows(p->nkb);
  prm.aug_blob = yy_layout ? p->aug_blob3 : p->aug_blob;
  prm.stats = p->stats;
  prm.pair_row = p->pair_row;
  prm.pair_cand = p->pair_cand;
  prm.max_pairs = p->max_pairs;
  prm.rowq = p->rowq;
  prm.ovf_rows = p->ovf_rows;
  prm.counters = p->counters;
  prm.metric = p->metric;
  prm.neg_mu_s = p->neg_mu_s;
  *out = prm;
  return cudaGetLastError();
}

cudaError_t tc_assign(TcPlan* p, const float* X, const float* C, const float* csq, uint32_t n,
                      uint32_t* result, uint32_t* assign, uint32_t* prev, uint32_t* d_changed, cudaStream_t st,
                      bool compute_csq) {
  using namespace tc;
  if (n > p->max_n) return cudaErrorInvalidValue;
  // TMA needs 16-byte aligned rows; the re-check kernels read both matrices with 16-byte vector loads
  if ((reinterpret_cast<uintptr_t>(X) & 15) || (reinterpret_cast<uintptr_t>(C) & 15)) return cudaErrorMisalignedAddress;
  cudaError_t e;
  Params prm;
  if ((e = tc_prepare(p, C, csq, n, &prm, st, false, compute_csq)) != cudaSuccess) return e;
  prm.X = X;
  prm.result = result;
  prm.assign = assign;      // non-null: the pass's bookkeeping (prev / assign / changed counter) is fused
  prm.prev = prev;
  prm.d_changed = d_changed;
  const unsigned grid = min(static_cast<uint32_t>(p->num_sms), prm.ntiles);
  const int slot = static_cast<int>(p->passes % TcPlan::kEvRing);
  if (p->capturing) {
    p->graph_slot = slot;
    cudaEventRecordWithFlags(p->ev0[slot], st, cudaEventRecordExternal);
  } else {
    p->graph_slot = -1;
    cudaEventRecord(p->ev0[slot], st);
  }
  tc_launch(0, false, p->nkb, grid, p->smem_bytes, st, p->tmap, prm);
  if (p->capturing) cudaEventRecordWithFlags(p->ev1[slot], st, cudaEventRecordExternal);
  else cudaEventRecord(p->ev1[slot], st);
  p->passes++;
  if ((e = cudaGetLastError()) != cudaSuccess) return e;
  // exact re-check of the multi-candidate rows, then the rows that need the full exact pass
  launch_recheck_pairs<0>(p->metric, p->num_sms * 4, st, X, C, csq, p->D, p->pair_row, p->pair_cand,
                          p->counters + CNT_PAIRS, p->max_pairs, n, p->K, p->pair_score);
  recheck_reduce_kernel<<<p->num_sms * 2, 256, 0, st>>>(p->rowq, p->counters + CNT_ROWQ, p->pair_cand,
                                                        p->pair_score, result, assign, prev, d_changed);
  if ((e = launch_assign_exact(p->metric, X, C, csq, n, p->D, p->K, p->ovf_rows, p->counters + CNT_OVF, result,
                               st)) != cudaSuccess)
    return e;
  if (assign)
    finalize_rows_kernel<<<p->num_sms, 256, 0, st>>>(p->ovf_rows, p->counters + CNT_OVF, result, assign, prev, d_changed);
  if ((e = cudaGetLastError()) != cudaSuccess) return e;
  if (p->inject_error) cudaMemsetAsync(p->counters + CNT_ERR, 0x11, sizeof(uint32_t), st);
  return cudaMemcpyAsync(p->h_counters, p->counters, sizeof(uint32_t) * CNT_N, cudaMemcpyDeviceToHost, st);
}

// resolves the positions of a row-list pass that took the exact list pass: result[i] = row_result[rows[i]]
__global__ void resolve_overflow_rows_kernel(const uint32_t* __restrict__ rows, uint32_t n,
                                             const uint32_t* __restrict__ row_result, uint32_t* __restrict__ result) {
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x)
    if (result[i] == kOverflowRow) result[i] = row_result[rows[i]];
}

cudaError_t tc_assign_rows(TcPlan* p, const float* X, uint32_t nX, const uint32_t* rows, uint32_t n, const float* C,
                           const float* csq, uint32_t* result, uint32_t* row_result, cudaStream_t st) {
  using namespace tc;
  if (n > p->max_n) return cudaErrorInvalidValue;
  if ((reinterpret_cast<uintptr_t>(X) & 15) || (reinterpret_cast<uintptr_t>(C) & 15)) return cudaErrorMisalignedAddress;
  cudaError_t e;
  Params prm;
  if ((e = tc_prepare(p, C, csq, n, &prm, st, false, true)) != cudaSuccess) return e;
  prm.X = X;
  prm.rows = rows;
  prm.result = result;
  const unsigned grid = min(static_cast<uint32_t>(p->num_sms), prm.ntiles);
  const int slot = static_cast<int>(p->passes % TcPlan::kEvRing);
  p->graph_slot = -1;
  cudaEventRecord(p->ev0[slot], st);
  tc_launch(0, true, p->nkb, grid, p->smem_bytes, st, p->tmap, prm);
  cudaEventRecord(p->ev1[slot], st);
  p->passes++;
  if ((e = cudaGetLastError()) != cudaSuccess) return e;
  launch_recheck_pairs<0>(p->metric, p->num_sms * 4, st, X, C, csq, p->D, p->pair_row, p->pair_cand,
                          p->counters + CNT_PAIRS, p->max_pairs, nX, p->K, p->pair_score);
  recheck_reduce_kernel<<<p->num_sms * 2, 256, 0, st>>>(p->rowq, p->counters + CNT_ROWQ, p->pair_cand,
                                                        p->pair_score, result, nullptr, nullptr, nullptr);
  if ((e = launch_assign_exact(p->metric, X, C, csq, n, p->D, p->K, p->ovf_rows, p->counters + CNT_OVF, row_result,
                               st)) != cudaSuccess)
    return e;
  resolve_overflow_rows_kernel<<<p->num_sms * 2, 256, 0, st>>>(rows, n, row_result, result);
  if ((e = cudaGetLastError()) != cudaSuccess) return e;
  if (p->inject_error) cudaMemsetAsync(p->counters + CNT_ERR, 0x11, sizeof(uint32_t), st);
  return cudaMemcpyAsync(p->h_counters, p->counters, sizeof(uint32_t) * CNT_N, cudaMemcpyDeviceToHost, st);
}

// Yinyang local step, candidate generation: for the listed rows, every centroid whose approximate score is
// within the rigorous margin of the row's second best, with its exact TRUE distance (reference
// METRIC::distance, metric_abstraction.h:59-101,179-222).  Results stay in the plan's queues (tc_queues()).
// Rows the filter cannot bound (NaN/Inf, > MAX_CAND candidates, queue full) are put on the overflow list.
cudaError_t tc_yy_candidates(TcPlan* p, const float* X, const float* C, const float* csq, uint32_t n,
                             const uint32_t* rows, const uint32_t* d_nrows, cudaStream_t st) {
  using namespace tc;
  if (n > p->max_n) return cudaErrorInvalidValue;
  if ((reinterpret_cast<uintptr_t>(X) & 15) || (reinterpret_cast<uintptr_t>(C) & 15)) return cudaErrorMisalignedAddress;
  cudaError_t e;
  Params prm;
  if ((e = tc_prepare(p, C, csq, n, &prm, st)) != cudaSuccess) return e;
  prm.X = X;
  prm.rows = rows;
  prm.d_nrows = d_nrows;
  const unsigned grid = min(static_cast<uint32_t>(p->num_sms), prm.ntiles);
  tc_launch(1, false, p->nkb, grid, p->smem_bytes, st, p->tmap, prm);
  if ((e = cudaGetLastError()) != cudaSuccess) return e;
  if ((e = tc_exact_distances(p, X, C, n, p->pair_row, p->pair_cand, p->counters + CNT_PAIRS, p->max_pairs,
                              p->pair_score, st)) != cudaSuccess)
    return e;
  return cudaMemcpyAsync(p->h_counters, p->counters, sizeof(uint32_t) * CNT_N, cudaMemcpyDeviceToHost, st);
}

// exact true distances of (row, centroid) pairs: 128 pairs per CTA, coalesced staging (see recheck_pairs_kernel)
cudaError_t tc_exact_distances(TcPlan* p, const float* X, const float* C, uint32_t n, const uint32_t* pair_row,
                               const uint32_t* pair_cand, const uint32_t* d_npairs, uint32_t max_pairs,
                               float* pair_score, cudaStream_t st) {
  launch_recheck_pairs<1>(p->metric, p->num_sms * 4, st, X, C, nullptr, p->D, pair_row, pair_cand, d_npairs, max_pairs,
                          n, p->K, pair_score);
  return cudaGetLastError();
}

// ---------------------------------------------------------------------------------------------------
// Yinyang bounds refresh on the tensor cores (reference kmeans_yy_init, kmeans.cu:431-485)
// ---------------------------------------------------------------------------------------------------
// exact part of the refresh: upper bound = distance to the own centroid, lower bound of the OWN group = nearest other
// member (both as the reference computes them).  Round 2's first version gave every sample a warp whose lanes each walked
// one member's row from global memory -- a chain of 256 dependent Kahan steps per lane with 10 of 32 lanes busy: 1.1 s
// at 8M x 256 @ 1024 (G = 102), more than the whole Lloyd run.  Now: (1) the (sample, group member) pairs of a chunk of
// rows are written to the plan's pair queue, (2) recheck_pairs_kernel computes their exact true distances (128 pairs
// per CTA, coalesced staging), (3) one thread per row folds its pairs into the two bounds.
__global__ void __launch_bounds__(256)
yy_own_pairs_kernel(uint32_t row0, uint32_t row1, uint32_t K, uint32_t G, const uint32_t* __restrict__ assign,
                    const uint32_t* __restrict__ groups, const uint32_t* __restrict__ goff,
                    const uint32_t* __restrict__ gmem, uint32_t* __restrict__ pair_row, uint32_t* __restrict__ pair_cand,
                    uint32_t max_pairs, uint32_t* __restrict__ rowq, uint32_t* __restrict__ counters) {
  const int lane = threadIdx.x & 31;
  const uint32_t stride = gridDim.x * blockDim.x;
  for (uint32_t base_row = row0 + blockIdx.x * blockDim.x; base_row < row1; base_row += stride) {
    const uint32_t row = base_row + threadIdx.x;
    uint32_t cnt = 0, beg = 0;
    if (row < row1) {
      const uint32_t a = assign[row];
      if (a < K) {                                   // "insane" samples keep FLT_MAX bounds
        const uint32_t g = groups[a];
        if (g < G) { beg = goff[g]; cnt = goff[g + 1] - beg; }
      }
    }
    uint32_t pre = cnt;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const uint32_t v = __shfl_up_sync(0xffffffffu, pre, o);
      if (lane >= o) pre += v;
    }
    const uint32_t warp_total = __shfl_sync(0xffffffffu, pre, 31);
    const unsigned have = __ballot_sync(0xffffffffu, cnt != 0);
    uint32_t pbase = 0, qbase = 0;
    if (lane == 0 && warp_total) {
      pbase = atomicAdd(&counters[tc::CNT_PAIRS], warp_total);
      qbase = atomicAdd(&counters[tc::CNT_ROWQ], static_cast<uint32_t>(__popc(have)));
    }
    pbase = __shfl_sync(0xffffffffu, pbase, 0) + (pre - cnt);
    qbase = __shfl_sync(0xffffffffu, qbase, 0) + __popc(have & ((1u << lane) - 1));
    if (cnt && pbase + cnt <= max_pairs) {           // (the host sizes the chunks so that this always holds)
      for (uint32_t j = 0; j < cnt; j++) {
        pair_row[pbase + j] = row;
        pair_cand[pbase + j] = gmem[beg + j];
      }
      rowq[3 * qbase] = row;
      rowq[3 * qbase + 1] = pbase;
      rowq[3 * qbase + 2] = cnt;
    } else if (cnt) {
      rowq[3 * qbase] = row;
      rowq[3 * qbase + 1] = 0;
      rowq[3 * qbase + 2] = 0;
    }
  }
}

__global__ void yy_own_reduce_kernel(const uint32_t* __restrict__ rowq, const uint32_t* __restrict__ d_nrowq,
                                     const uint32_t* __restrict__ pair_cand, const float* __restrict__ pair_score,
                                     const uint32_t* __restrict__ assign, const uint32_t* __restrict__ groups, uint32_t G,
                                     float* __restrict__ bounds) {
  const uint32_t nq = *d_nrowq;
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < nq; i += gridDim.x * blockDim.x) {
    const uint32_t row = rowq[3 * i], base = rowq[3 * i + 1], cnt = rowq[3 * i + 2];
    if (cnt == 0) continue;
    const uint32_t a = assign[row];
    float lb = FLT_MAX, ub = FLT_MAX;
    for (uint32_t j = 0; j < cnt; j++) {
      const float d = pair_score[base + j];
      if (pair_cand[base + j] == a) ub = d;
      else if (d < lb) lb = d;                       // NaN never lowers a bound (as the reference's `dist < bound`)
    }
    float* b = bounds + static_cast<size_t>(row) * (G + 1);
    b[0] = ub;
    b[1 + groups[a]] = lb;
  }
}

// Builds the group-sorted table layout from the centroid -> group map of this run (host vector, G groups; ids >= G
// mark dead centroids, which get no table row).  Call again whenever the grouping changes.
void tc_yy_layout_host(const uint32_t* host_groups, uint32_t K, uint32_t G, std::vector<uint32_t>* perm_out,
                       std::vector<uint32_t>* qgroup_out, std::vector<uint32_t>* goff_out,
                       std::vector<uint32_t>* gmem_out, int* nt3_out) {
  using namespace tc;
  std::vector<uint32_t> gsz(G, 0);
  for (uint32_t c = 0; c < K; c++)
    if (host_groups[c] < G) gsz[host_groups[c]]++;
  std::vector<uint32_t> goff(G + 1, 0), gfill(G, 0), gmem(K ? K : 1, 0);
  for (uint32_t g = 0; g < G; g++) goff[g + 1] = goff[g] + gsz[g];
  for (uint32_t c = 0; c < K; c++)
    if (host_groups[c] < G) gmem[goff[host_groups[c]] + gfill[host_groups[c]]++] = c;
  size_t rows = 0;
  for (uint32_t g = 0; g < G; g++) rows += (gsz[g] + 3) / 4 * 4;
  const int nt3 = static_cast<int>(std::max<size_t>(1, (rows + TN - 1) / TN));
  const size_t rows_pad = static_cast<size_t>(nt3) * TN;
  std::vector<uint32_t> perm(rows_pad, UINT32_MAX), qgroup(rows_pad / 4, UINT32_MAX);
  size_t r = 0;
  for (uint32_t g = 0; g < G; g++) {
    if (gsz[g] == 0) continue;
    for (uint32_t j = 0; j < gsz[g]; j++) perm[r + j] = gmem[goff[g] + j];
    const size_t padded = (gsz[g] + 3) / 4 * 4;
    for (size_t qd = r / 4; qd < (r + padded) / 4; qd++) qgroup[qd] = g;
    r += padded;
  }
  *perm_out = std::move(perm);
  *qgroup_out = std::move(qgroup);
  *goff_out = std::move(goff);
  *gmem_out = std::move(gmem);
  *nt3_out = nt3;
}

cudaError_t tc_yy_layout(TcPlan* p, const uint32_t* host_groups, uint32_t G) {
  using namespace tc;
  std::vector<uint32_t> perm, qgroup, goff, gmem;
  int nt3 = 0;
  tc_yy_layout_host(host_groups, p->K, G, &perm, &qgroup, &goff, &gmem, &nt3);
  const size_t rows_pad = static_cast<size_t>(nt3) * TN;
  cudaError_t e;
  if (nt3 != p->nt3 || !p->table3) {
    pool_free(p->table3); pool_free(p->aug_blob3); pool_free(p->yy_perm); pool_free(p->yy_qgroup);
    p->table3 = nullptr; p->aug_blob3 = nullptr; p->yy_perm = nullptr; p->yy_qgroup = nullptr;
    if ((e = pool_alloc(reinterpret_cast<void**>(&p->table3), rows_pad * p->nkb * KB * sizeof(__half))) != cudaSuccess) return e;
    if ((e = pool_alloc(reinterpret_cast<void**>(&p->aug_blob3), static_cast<size_t>(nt3) * AUG_B_BYTES)) != cudaSuccess) return e;
    if ((e = pool_alloc(reinterpret_cast<void**>(&p->yy_perm), rows_pad * sizeof(uint32_t))) != cudaSuccess) return e;
    if ((e = pool_alloc(reinterpret_cast<void**>(&p->yy_qgroup), rows_pad / 4 * sizeof(uint32_t))) != cudaSuccess) return e;
    if ((e = encode_table_map(&p->tmap3, p->table3, rows_pad, p->nkb)) != cudaSuccess) return e;
    p->nt3 = nt3;
  }
  if (G != p->G3 || !p->yy_goff) {
    pool_free(p->yy_goff); pool_free(p->yy_gmem);
    p->yy_goff = nullptr; p->yy_gmem = nullptr;
    if ((e = pool_alloc(reinterpret_cast<void**>(&p->yy_goff), (static_cast<size_t>(G) + 1) * sizeof(uint32_t))) != cudaSuccess) return e;
    if ((e = pool_alloc(reinterpret_cast<void**>(&p->yy_gmem), gmem.size() * sizeof(uint32_t))) != cudaSuccess) return e;
    p->G3 = G;
  }
  p->yy_max_gsize = 0;
  for (uint32_t g = 0; g < G; g++) p->yy_max_gsize = std::max(p->yy_max_gsize, goff[g + 1] - goff[g]);
  if ((e = cudaMemcpy(p->yy_perm, perm.data(), perm.size() * 4, cudaMemcpyHostToDevice)) != cudaSuccess) return e;
  if ((e = cudaMemcpy(p->yy_qgroup, qgroup.data(), qgroup.size() * 4, cudaMemcpyHostToDevice)) != cudaSuccess) return e;
  if ((e = cudaMemcpy(p->yy_goff, goff.data(), goff.size() * 4, cudaMemcpyHostToDevice)) != cudaSuccess) return e;
  return cudaMemcpy(p->yy_gmem, gmem.data(), gmem.size() * 4, cudaMemcpyHostToDevice);
}

bool tc_yy_layout_ready(TcPlan* p, uint32_t G) { return p && p->table3 && p->G3 == G; }

// One bounds refresh: bounds[row] = {ub exact, lb[g] valid lower bounds} (see Params, MODE 3).  Rows the filter
// cannot bound are left on the overflow list (tc_queues) for the caller's exact row refresh.
cudaError_t tc_yy_refresh(TcPlan* p, const float* X, const float* C, const float* csq, uint32_t n,
                          const uint32_t* assign, const uint32_t* groups, uint32_t G, float* bounds, cudaStream_t st) {
  using namespace tc;
  if (n > p->max_n || !tc_yy_layout_ready(p, G)) return cudaErrorInvalidValue;
  if ((reinterpret_cast<uintptr_t>(X) & 15) || (reinterpret_cast<uintptr_t>(C) & 15)) return cudaErrorMisalignedAddress;
  cudaError_t e;
  if ((e = launch_fill_u32(reinterpret_cast<uint32_t*>(bounds), 0x7f7fffffu /* FLT_MAX */,
                           static_cast<size_t>(n) * (G + 1), st)) != cudaSuccess)
    return e;
  Params prm;
  if ((e = tc_prepare(p, C, csq, n, &prm, st, true)) != cudaSuccess) return e;
  prm.yy_qgroup = p->yy_qgroup;
  prm.yy_groups = groups;
  prm.yy_assign = assign;
  prm.yy_bounds = bounds;
  prm.G = G;
  prm.X = X;
  const unsigned grid = min(static_cast<uint32_t>(p->num_sms), prm.ntiles);
  tc_launch(3, false, p->nkb, grid, p->smem_bytes, st, p->tmap3, prm);
  if ((e = cudaGetLastError()) != cudaSuccess) return e;
  // own group + upper bound, exactly: chunks of rows whose pairs fit the queue (yy_max_gsize members per row at most)
  const uint32_t per_row = max(1u, p->yy_max_gsize);
  const uint32_t chunk = max(1u, p->max_pairs / per_row);
  for (uint32_t r0 = 0; r0 < n; r0 += chunk) {
    const uint32_t r1 = min(n, r0 + chunk);
    if ((e = cudaMemsetAsync(p->counters, 0, sizeof(uint32_t) * 2, st)) != cudaSuccess) return e;   // CNT_PAIRS, CNT_ROWQ
    yy_own_pairs_kernel<<<p->num_sms * 8, 256, 0, st>>>(r0, r1, p->K, G, assign, groups, p->yy_goff, p->yy_gmem, p->pair_row,
                                                       p->pair_cand, p->max_pairs, p->rowq, p->counters);
    if ((e = tc_exact_distances(p, X, C, n, p->pair_row, p->pair_cand, p->counters + CNT_PAIRS, p->max_pairs,
                                p->pair_score, st)) != cudaSuccess)
      return e;
    yy_own_reduce_kernel<<<p->num_sms * 4, 256, 0, st>>>(p->rowq, p->counters + CNT_ROWQ, p->pair_cand, p->pair_score, assign,
                                                        groups, G, bounds);
  }
  if ((e = cudaGetLastError()) != cudaSuccess) return e;
  return cudaMemcpyAsync(p->h_counters, p->counters, sizeof(uint32_t) * CNT_N, cudaMemcpyDeviceToHost, st);
}

void tc_queues(TcPlan* p, TcQueues* q) {
  q->rowq = p->rowq;
  q->d_nrowq = p->counters + tc::CNT_ROWQ;
  q->pair_cand = p->pair_cand;
  q->pair_score = p->pair_score;
  q->ovf_rows = p->ovf_rows;
  q->d_novf = p->counters + tc::CNT_OVF;
}

// valid after the stream has been synchronised
void tc_last_stats(TcPlan* p, uint32_t* n_recheck, uint32_t* n_overflow) {
  *n_recheck = p->h_counters[tc::CNT_ROWQ];
  *n_overflow = p->h_counters[tc::CNT_OVF];
}

uint32_t tc_last_error(TcPlan* p) { return p->h_counters[tc::CNT_ERR]; }
void tc_set_capture(TcPlan* p, bool on) { p->capturing = on; }
uint32_t tc_last_pairs(TcPlan* p) { return p->h_counters[tc::CNT_PAIRS]; }

// device time (ms) of the main kernel in the most recent passes, oldest first; call after a sync
int tc_kernel_times(TcPlan* p, float* ms_out, int max_out) {
  const uint64_t have = p->passes < static_cast<uint64_t>(TcPlan::kEvRing) ? p->passes : TcPlan::kEvRing;
  const int n = static_cast<int>(have < static_cast<uint64_t>(max_out) ? have : max_out);
  for (int i = 0; i < n; i++) {
    // graph replays refresh the one slot that was captured; otherwise the ring holds one pair per pass
    const int slot = p->graph_slot >= 0 ? p->graph_slot : static_cast<int>((p->passes - n + i) % TcPlan::kEvRing);
    float ms = 0.f;
    if (cudaEventElapsedTime(&ms, p->ev0[slot], p->ev1[slot]) != cudaSuccess) ms = -1.f;
    ms_out[i] = ms;
  }
  return n;
}

// ===================================================================================================
// k-NN on the tensor cores (reference knn.cu:177-347: cluster-pruned exact k nearest neighbours)
//
// Queries and candidates are the samples in cluster-sorted order (the inverse assignment).  Pass 1 multiplies
// every query tile (<= 128 queries of one cluster) with the blocks covering its own cluster; that yields, per
// query, an upper bound of the distance to its k-th neighbour.  The reference's skip test
// `Cd[B][A] - d(q, A) - R[B] > kth` (knn.cu:218-225) is then evaluated per tile (a cluster is visited if ANY
// query of the tile needs it) and pass 2 visits the surviving clusters' blocks.  The epilogue records every
// column whose fp16 score is within the rigorous margin of the row's (k+1)-th best (self included); those
// candidates get their exact distance (reference METRIC::distance) and the k smallest are written in
// ascending order.  Any superset of the reference's visited clusters gives the same exact top-k.
// ===================================================================================================
namespace knn {

__global__ void tile_count_kernel(const uint32_t* __restrict__ off, uint32_t K, uint32_t* __restrict__ ntile) {
  uint32_t c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c < K) ntile[c] = (off[c + 1] - off[c] + tc::TM - 1) / tc::TM;
}

// per cluster: its blocks (= query tiles), the two own-cluster segments of pass 1
__global__ void tile_fill_kernel(const uint32_t* __restrict__ off, uint32_t K, const uint32_t* __restrict__ blk_first,
                                 uint32_t* __restrict__ tile_nrows, uint32_t* __restrict__ blk_cluster,
                                 uint2* __restrict__ ranges1, uint32_t* __restrict__ roff1,
                                 uint32_t* __restrict__ rcount1, uint32_t* __restrict__ nblk1,
                                 uint32_t* __restrict__ d_ntiles, unsigned long long* __restrict__ d_pairs) {
  uint32_t c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= K) return;
  const uint32_t m = off[c + 1] - off[c];
  const uint32_t t0 = blk_first[c], nt = (m + tc::TM - 1) / tc::TM;
  for (uint32_t i = 0; i < nt; i++) {
    const uint32_t t = t0 + i;
    tile_nrows[t] = min(static_cast<uint32_t>(tc::TM), m - i * tc::TM);
    blk_cluster[t] = c;
    ranges1[2 * t] = ranges1[2 * t + 1] = make_uint2(t0, t0 + nt - 1);   // threshold sweep + recording sweep
    roff1[t] = 2 * t;
    rcount1[t] = 2;
    nblk1[t] = 2 * nt;
  }
  if (c == K - 1) *d_ntiles = t0 + nt;
}

// table row of every valid sorted position (cluster-aligned, zero padded): tab2orig[row] = original sample index
__global__ void layout_kernel(const uint32_t* __restrict__ inv, const uint32_t* __restrict__ assign,
                              const uint32_t* __restrict__ off, const uint32_t* __restrict__ blk_first, uint32_t nv,
                              uint32_t* __restrict__ tab2orig) {
  uint32_t pos = blockIdx.x * blockDim.x + threadIdx.x;
  if (pos >= nv) return;
  const uint32_t s = inv[pos], c = assign[s];
  tab2orig[blk_first[c] * tc::TM + (pos - off[c])] = s;
}

// one warp per table row: ||y - c||^2 (fp32) and the largest s-free magnitude |y| + |c| (for the centring error)
__global__ void prep_norms_kernel(const float* __restrict__ X, const float* __restrict__ C, int D,
                                  const uint32_t* __restrict__ tab2orig, const uint32_t* __restrict__ blk_cluster,
                                  const uint32_t* __restrict__ d_ntiles, float* __restrict__ ysq,
                                  float* __restrict__ yabs_max, int angular) {
  const uint32_t row = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (row >= *d_ntiles * tc::TM) return;
  const uint32_t sidx = tab2orig[row];
  if (sidx == UINT32_MAX) {
    if (lane == 0) ysq[row] = 0.f;
    return;
  }
  const float* x = X + static_cast<size_t>(sidx) * D;
  const float* c = C + static_cast<size_t>(blk_cluster[row / tc::TM]) * D;
  float a = 0.f, r = 0.f;
  for (int f = lane; f < D; f += 32) {
    const float xv = x[f], cv = c[f], d = xv - cv, m = fabsf(xv) + fabsf(cv);
    a = fmaf(d, d, a);
    r = fmaf(m, m, r);
  }
  for (int o = 16; o > 0; o >>= 1) {
    a += __shfl_xor_sync(0xffffffffu, a, o);
    r += __shfl_xor_sync(0xffffffffu, r, o);
  }
  if (lane == 0) {
    ysq[row] = a;
    if (r == r && r < 3.0e38f) atomicMax(reinterpret_cast<uint32_t*>(yabs_max), __float_as_uint(__fsqrt_ru(r)));
  }
  if (angular) {   // deviation of the sample from unit length (yabs_max[1]); NaN / Inf rows count as "far off"
    float xx = 0.f;
    for (int f = lane; f < D; f += 32) xx = fmaf(x[f], x[f], xx);
    for (int o = 16; o > 0; o >>= 1) xx += __shfl_xor_sync(0xffffffffu, xx, o);
    const float dev = fabsf(xx - 1.f) + 4.0e-6f * (1.f + xx);    // + the fp32 rounding of the sum itself
    if (lane == 0) atomicMax(reinterpret_cast<uint32_t*>(yabs_max + 1), (dev == dev) ? __float_as_uint(dev) : 0x7f800000u);
  }
}

// one warp per table row: fp16(s (y - c)), rounding residual, bias -(s^2 |y - c|^2 / 2) in three fp16 terms;
// padding and non-finite rows: zero vector, bias -65504
__global__ void prep_table_kernel(const float* __restrict__ X, const float* __restrict__ C, int D, int nkb,
                                  const uint32_t* __restrict__ tab2orig, const uint32_t* __restrict__ blk_cluster,
                                  const uint32_t* __restrict__ d_ntiles, const float* __restrict__ ysq,
                                  __half* __restrict__ table, __half* __restrict__ aug_blob,
                                  tc::Stats* __restrict__ st, const float* __restrict__ yabs_max, int angular,
                                  uint32_t* __restrict__ d_error) {
  using namespace tc;
  const uint32_t row = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (row >= *d_ntiles * TM) return;
  const int Dp = nkb * KB;
  const float s = st->scale;
  if (row == 0 && lane == 0) {
    st->yabs = *yabs_max * s * 1.0001f;
    st->knn_extra = 0.f;
    if (angular) {
      // angular neighbours through the L2 pass: for |1 - |y|^2| <= eps the true top-k by dot product lie within
      // s^2 * eps of the (k+1)-th best L2 score (x.y = (|x|^2 + |y|^2 - d^2) / 2), so the margin grows by that much;
      // samples far from unit length make the equivalence useless -> the caller runs the exact search instead
      const float eps = yabs_max[1];
      if (!(eps <= 1.0e-2f)) *d_error = 2u;
      st->knn_extra = (s * s) * eps * 1.01f;
    }
  }
  const uint32_t sidx = tab2orig[row];
  bool finite = sidx != UINT32_MAX;
  const float* x = X + static_cast<size_t>(finite ? sidx : 0) * D;
  const float* c = C + static_cast<size_t>(blk_cluster[row / TM]) * D;
  if (finite) {
    const float q = ysq[row];
    finite = (q == q) && q < 3.0e38f;
    finite = __all_sync(0xffffffffu, finite);
  }
  float d2 = 0.f;
  for (int f = lane; f < Dp; f += 32) {
    const float v = (finite && f < D) ? (x[f] - c[f]) * s : 0.f;
    const __half h = __float2half_rn(v);
    const float r = v - __half2float(h);
    d2 = fmaf(r, r, d2);
    table[static_cast<size_t>(row) * Dp + f] = h;
  }
  for (int o = 16; o > 0; o >>= 1) d2 += __shfl_xor_sync(0xffffffffu, d2, o);
  if (lane == 0) {
    if (finite) atomicMax(reinterpret_cast<uint32_t*>(&st->dcmax), __float_as_uint(__fsqrt_ru(d2) * 1.0001f));
    write_bias_row(aug_blob, row, finite, finite ? -0.5f * ((s * ysq[row]) * s) : 0.f);
  }
}

// one warp per tile: the clusters pass 2 must visit, one segment (block range) per cluster.  P = parts per row of the
// candidate pass (2; 4 on 64-row tiles): the tightest of the parts' bounds is the row's
template <int P>
__global__ void __launch_bounds__(256)
range_build_kernel(const uint32_t* __restrict__ d_ntiles, const uint32_t* __restrict__ tile_nrows,
                   const uint32_t* __restrict__ blk_cluster, const uint32_t* __restrict__ blk_first,
                   const uint32_t* __restrict__ off, uint32_t K, const float* __restrict__ cd,
                   const float* __restrict__ radii, const float* __restrict__ ysq, const float* __restrict__ dub,
                   uint2* __restrict__ pool, uint32_t pool_cap, uint32_t* __restrict__ pool_used,
                   uint32_t* __restrict__ roff2, uint32_t* __restrict__ rcount2, uint32_t* __restrict__ nblk2,
                   uint32_t* __restrict__ d_error, unsigned long long* __restrict__ d_pairs, uint32_t part,
                   uint32_t nparts) {
  const int lane = threadIdx.x & 31;
  const uint32_t warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, nwarps = (gridDim.x * blockDim.x) >> 5;
  const uint32_t T = *d_ntiles;
  const uint32_t t_lo = static_cast<uint32_t>(static_cast<uint64_t>(T) * part / nparts);
  const uint32_t t_hi = static_cast<uint32_t>(static_cast<uint64_t>(T) * (part + 1) / nparts);
  for (uint32_t t = t_lo + warp; t < t_hi; t += nwarps) {
    const uint32_t nr = tile_nrows[t], A = blk_cluster[t];
    // W = max over the tile's queries of d(q, A) + (upper bound of the distance to the k-th neighbour so far);
    // d(q, A) is bounded by the fp32 centred norm (the reference's Kahan value differs by rounding only)
    float W = 0.f;
    for (uint32_t r = lane; r < nr; r += 32) {
      const uint32_t row = t * tc::TM + r;
      float ub = dub[P * row];
#pragma unroll
      for (int q = 1; q < P; q++) ub = fminf(ub, dub[P * row + q]);
      const float w = __fsqrt_ru(ysq[row]) * 1.00001f + ub;
      W = (w == w) ? fmaxf(W, w) : INFINITY;
    }
    for (int o = 16; o > 0; o >>= 1) W = fmaxf(W, __shfl_xor_sync(0xffffffffu, W, o));
    W = W * 1.000002f + 1e-30f;   // the reference rounds `cd - dA - R` twice: stay on the visiting side
    for (int pass = 0; pass < 2; pass++) {   // pass 0 counts, pass 1 writes
      uint32_t count = 0, blocks = 0, base = 0;
      unsigned long long pairs = 0;
      if (pass == 0 && lane == 0 && A < K) pairs = static_cast<unsigned long long>(nr) * (off[A + 1] - off[A]);   // own cluster
      if (pass == 1) {
        const uint32_t c0 = rcount2[t];
        if (lane == 0) base = atomicAdd(pool_used, c0);
        base = __shfl_sync(0xffffffffu, base, 0);
        if (base + c0 > pool_cap) {
          if (lane == 0) { *d_error = 1u; rcount2[t] = 0; nblk2[t] = 0; roff2[t] = 0; }
          break;
        }
        if (lane == 0) roff2[t] = base;
      }
      for (uint32_t B0 = 0; B0 < K; B0 += 32) {
        const uint32_t B = B0 + lane;
        bool visit = false;
        uint32_t lo = 0, hi = 0;
        if (B < K && B != A) {
          const uint32_t m = off[B + 1] - off[B];
          const float c = cd[static_cast<size_t>(B) * K + A];
          if (m && c == c && !(c - radii[B] > W)) {
            visit = true;
            lo = blk_first[B];
            hi = blk_first[B + 1] - 1;
            pairs += static_cast<unsigned long long>(m) * nr;
          }
        }
        const unsigned mk = __ballot_sync(0xffffffffu, visit);
        if (visit) {
          if (pass == 1) pool[base + count + __popc(mk & ((1u << lane) - 1))] = make_uint2(lo, hi);
        }
        uint32_t nb = visit ? hi - lo + 1 : 0;
        for (int o = 16; o > 0; o >>= 1) nb += __shfl_xor_sync(0xffffffffu, nb, o);
        blocks += nb;
        count += __popc(mk);
      }
      if (pass == 0) {
        if (lane == 0) { rcount2[t] = count; nblk2[t] = blocks; }
        for (int o = 16; o > 0; o >>= 1) pairs += __shfl_xor_sync(0xffffffffu, pairs, o);
        if (lane == 0 && pairs) atomicAdd(d_pairs, pairs);
        __syncwarp();
      }
    }
  }
}

// one warp per query (table row): final threshold, expansion of the recorded entries into candidate pairs.  P = parts
// per row (2 halves; 4 quarters on 64-row tiles), whose lists are merged here
template <int P>
__global__ void __launch_bounds__(256)
expand_kernel(const uint32_t* __restrict__ d_ntiles, int kk, uint32_t stride, const float* __restrict__ topk,
              const uint32_t* __restrict__ cnts, const uint32_t* __restrict__ flags,
              const uint4* __restrict__ entries, const uint32_t* __restrict__ tab2orig, uint32_t max_pairs,
              uint32_t* __restrict__ pair_row, uint32_t* __restrict__ pair_cand, uint32_t* __restrict__ rowq,
              uint32_t* __restrict__ fb_rows, uint32_t* __restrict__ counters, uint32_t* __restrict__ dbg,
              uint32_t part, uint32_t nparts) {
  const int lane = threadIdx.x & 31;
  const uint32_t warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, nwarps = (gridDim.x * blockDim.x) >> 5;
  const uint32_t T = *d_ntiles;
  const uint32_t row_lo = static_cast<uint32_t>(static_cast<uint64_t>(T) * part / nparts) * tc::TM;
  const uint32_t nrows = static_cast<uint32_t>(static_cast<uint64_t>(T) * (part + 1) / nparts) * tc::TM;
  for (uint32_t row = row_lo + warp; row < nrows; row += nwarps) {
    const uint32_t self = tab2orig[row];
    if (self == UINT32_MAX) continue;   // padding
    const uint32_t s0 = P * row;
    float kq[P];
#pragma unroll
    for (int q = 0; q < P; q++) kq[q] = topk[static_cast<size_t>(kk - 1) * stride + s0 + q];
    float kth = kq[0];   // each part saw kk distinct columns at or above its own value
#pragma unroll
    for (int q = 1; q < P; q++) kth = fmaxf(kth, kq[q]);
    uint32_t fl = flags[s0], cs[P];
#pragma unroll
    for (int q = 1; q < P; q++) fl |= flags[s0 + q];
#pragma unroll
    for (int q = 0; q < P; q++) cs[q] = cnts[s0 + q];
    // entry i of the concatenated (part 0, part 1, ...) lists
    auto entry = [&](uint32_t i) {
      if constexpr (P == 2)
        return i < cs[0] ? entries[static_cast<size_t>(s0) * tc::KNN_CAP + i]
                         : entries[static_cast<size_t>(s0 + 1) * tc::KNN_CAP + (i - cs[0])];
      uint32_t s = s0;
#pragma unroll
      for (int q = 0; q < P - 1; q++)
        if (s == s0 + q && i >= cs[q]) { i -= cs[q]; s++; }
      return entries[static_cast<size_t>(s) * tc::KNN_CAP + i];
    };
    bool fallback = fl != 0 || !(kth > -INFINITY);
    if (lane == 0 && dbg) {
      if (fl & 1) atomicAdd(dbg + 0, 1u);
      if (fl & 2) atomicAdd(dbg + 1, 1u);
      if (fl & 4) atomicAdd(dbg + 2, 1u);
      if (!(kth > -INFINITY)) atomicAdd(dbg + 3, 1u);
    }
    // each lane takes entries lane, lane+32, ... of the concatenated lists; an entry survives if its group maximum is
    // within ITS margin of the final kk-th best
    uint32_t mine = 0, total_e = 0;
#pragma unroll
    for (int q = 0; q < P; q++) total_e += cs[q];
    for (uint32_t i = lane; i < total_e && !fallback; i += 32) {
      const uint4 e = entry(i);
      if (__uint_as_float(e.x) >= kth - __uint_as_float(e.w)) {
        uint32_t m = e.y;
        const uint32_t p0 = (e.z >> 2) * 128u + ((e.z >> 1) & 1u) * 64u + (e.z & 1u) * 32u;
        while (m) {
          const uint32_t cp = p0 + __ffs(m) - 1;
          m &= m - 1;
          if (cp != row && tab2orig[cp] != UINT32_MAX) mine++;
        }
      }
    }
    uint32_t pre = mine;
    for (int o = 1; o < 32; o <<= 1) {
      uint32_t v = __shfl_up_sync(0xffffffffu, pre, o);
      if (lane >= o) pre += v;
    }
    const uint32_t total = __shfl_sync(0xffffffffu, pre, 31);
    if (lane == 0 && dbg && !fallback) {
      if (total > 64) atomicAdd(dbg + 4, 1u);
      if (total < static_cast<uint32_t>(kk - 1)) atomicAdd(dbg + 5, 1u);
      atomicAdd(dbg + 6, total);
    }
    if (total > 64 || total < static_cast<uint32_t>(kk - 1)) fallback = true;
    uint32_t base = 0;
    if (!fallback) {
      if (lane == 0) base = atomicAdd(&counters[tc::CNT_PAIRS], total);
      base = __shfl_sync(0xffffffffu, base, 0);
      if (base + total > max_pairs) fallback = true;
    }
    if (fallback) {
      if (lane == 0) fb_rows[atomicAdd(&counters[tc::CNT_OVF], 1u)] = self;
      continue;
    }
    uint32_t w = base + pre - mine;
    for (uint32_t i = lane; i < total_e; i += 32) {
      const uint4 e = entry(i);
      if (__uint_as_float(e.x) >= kth - __uint_as_float(e.w)) {
        uint32_t m = e.y;
        const uint32_t p0 = (e.z >> 2) * 128u + ((e.z >> 1) & 1u) * 64u + (e.z & 1u) * 32u;
        while (m) {
          const uint32_t cp = p0 + __ffs(m) - 1;
          m &= m - 1;
          const uint32_t o = tab2orig[cp];
          if (cp != row && o != UINT32_MAX) {
            pair_row[w] = self;
            pair_cand[w] = o;
            w++;
          }
        }
      }
    }
    if (lane == 0) {
      const uint32_t q = atomicAdd(&counters[tc::CNT_ROWQ], 1u);
      rowq[3 * q] = self;
      rowq[3 * q + 1] = base;
      rowq[3 * q + 2] = total;
    }
  }
}

// one warp per query: the k smallest exact distances in ascending order (knn.cu:239-242)
__global__ void __launch_bounds__(256)
select_kernel(int k, const uint32_t* __restrict__ rowq, const uint32_t* __restrict__ counters,
              const uint32_t* __restrict__ pair_cand, const float* __restrict__ pair_score, uint32_t q_offset,
              uint32_t* __restrict__ neighbors) {
  const int lane = threadIdx.x & 31;
  const uint32_t warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, nwarps = (gridDim.x * blockDim.x) >> 5;
  const uint32_t nq = counters[tc::CNT_ROWQ];
  for (uint32_t q = warp; q < nq; q += nwarps) {
    const uint32_t row = rowq[3 * q], base = rowq[3 * q + 1], cnt = rowq[3 * q + 2];
    float d[2];
    uint32_t id[2];
#pragma unroll
    for (int j = 0; j < 2; j++) {
      const uint32_t i = lane + 32 * j;
      d[j] = INFINITY;
      id[j] = UINT32_MAX;
      if (i < cnt) {
        const float v = pair_score[base + i];
        if (v == v) { d[j] = v; id[j] = pair_cand[base + i]; }
      }
    }
    for (int r = 0; r < k; r++) {
      // lexicographic (distance, index) minimum over the 64 slots
      float bd = d[0];
      uint32_t bi = id[0];
      if (d[1] < bd || (d[1] == bd && id[1] < bi)) { bd = d[1]; bi = id[1]; }
      for (int o = 16; o > 0; o >>= 1) {
        const float od = __shfl_xor_sync(0xffffffffu, bd, o);
        const uint32_t oi = __shfl_xor_sync(0xffffffffu, bi, o);
        if (od < bd || (od == bd && oi < bi)) { bd = od; bi = oi; }
      }
      if (lane == 0) neighbors[static_cast<size_t>(row - q_offset) * k + r] = bi;
      if (id[0] == bi) { d[0] = INFINITY; id[0] = UINT32_MAX; }
      if (id[1] == bi) { d[1] = INFINITY; id[1] = UINT32_MAX; }
    }
  }
}

}  // namespace knn

bool tc_knn_supported(int metric, int k, uint32_t N, int D, uint32_t K) {
  // (the angular metric is served through the L2 pass when the samples have unit length, see tc_knn_search)
  if (k + 1 > tc::KNN_MAX_KK) return false;
  if (D < 4 || D % 4 != 0 || D > tc::MAX_TILE64_NKB * tc::KB) return false;   // D > 512: 64-row tiles
  if (N < 4096 || N > (1u << 30)) return false;                    // tiny inputs: not worth the set-up
  if (static_cast<uint64_t>(K) * K > (1ull << 31)) return false;
  return true;
}

#define KNN_TRY(x) do { e = (x); if (e != cudaSuccess) goto done; } while (0)

// neighbors: device array [N][k] indexed by the original sample index (this build shards k-NN queries only on the
// SIMT path).  Rows the filter cannot serve are appended to fb_rows / d_nfb for the caller's exact search.
cudaError_t tc_knn_search(int metric, int k, const float* X, const float* C, uint32_t N, int D, uint32_t K,
                          const uint32_t* assign, const uint32_t* inv, const uint32_t* off, const float* cd,
                          const float* radii, uint32_t nv, uint32_t* neighbors, uint32_t* fb_rows, uint32_t* d_nfb,
                          unsigned long long* d_pairs, uint32_t* h_error, uint32_t part, uint32_t nparts,
                          cudaStream_t st) {
  using namespace tc;
  cudaError_t e = cudaSuccess;
  *h_error = 0;
  int dev = 0, num_sms = 132;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&num_sms, cudaDevAttrMultiProcessorCount, dev);
  const int nkb = (D + KB - 1) / KB, kk = k + 1;
  const uint32_t tmax = nv / TM + K + 1;                 // upper bound of the number of cluster-aligned blocks
  const uint32_t rows_max = tmax * TM;
  // per-part state of the candidate pass: a row has two 64-column halves, or four 32-column parts on the 64-row tiles
  // of D > 512 (tc_assign_body); range_build_kernel / expand_kernel merge the parts of a row
  const bool t64 = tile64(nkb);
  const uint32_t stride = (t64 ? 4u : 2u) * rows_max;
  const uint64_t want_pool = static_cast<uint64_t>(tmax) * K;
  const uint32_t pool_cap = static_cast<uint32_t>(want_pool < (48u << 20) ? want_pool : (48u << 20));
  const uint32_t pair_cap = static_cast<uint32_t>(std::min<uint64_t>(40ull * nv + 4096, 0xFFFFFFF0ull));
  __half *table = nullptr, *blobs = nullptr;
  float *ysq = nullptr, *topk = nullptr, *dub = nullptr, *pair_score = nullptr, *yabs = nullptr;
  Stats* stats = nullptr;
  uint32_t *u32 = nullptr, *kcnt = nullptr, *kflags = nullptr, *pair_row = nullptr, *pair_cand = nullptr, *rowq = nullptr;
  uint32_t *counters = nullptr, *tab2orig = nullptr;
  uint2 *ranges1 = nullptr, *pool = nullptr;
  uint4* entries = nullptr;
  void* cub_tmp = nullptr;
  size_t cub_bytes = 0;
  uint32_t h_cnt[CNT_N + 2] = {0};
  uint32_t h_dbg[8] = {0};
  CUtensorMap tmap;
  Params prm;
  const unsigned grid = static_cast<unsigned>(num_sms);
  const size_t smem_bytes = smem_layout(nkb).total + 1024;
  uint32_t *ntile, *blk_first, *t_nrows, *blk_cluster, *roff1, *rcount1, *nblk1, *roff2, *rcount2, *nblk2, *d_ntiles,
      *pool_used, *d_err;
  {
    const size_t words = static_cast<size_t>(K) + (K + 1) + 8ull * tmax + 16;
    KNN_TRY(pool_alloc(reinterpret_cast<void**>(&u32), words * sizeof(uint32_t)));
    KNN_TRY(cudaMemsetAsync(u32, 0, words * sizeof(uint32_t), st));
    uint32_t* q = u32;
    ntile = q; q += K;
    blk_first = q; q += K + 1;
    t_nrows = q; q += tmax; blk_cluster = q; q += tmax;
    roff1 = q; q += tmax; rcount1 = q; q += tmax; nblk1 = q; q += tmax;
    roff2 = q; q += tmax; rcount2 = q; q += tmax; nblk2 = q; q += tmax;
    d_ntiles = q++; pool_used = q++; d_err = q++;   // pool_used + 2 .. + 9: debug counters of expand_kernel
  }
  KNN_TRY(pool_alloc(reinterpret_cast<void**>(&table), static_cast<size_t>(rows_max) * nkb * KB * sizeof(__half)));
  KNN_TRY(pool_alloc(reinterpret_cast<void**>(&blobs), static_cast<size_t>(tmax) * AUG_B_BYTES));
  KNN_TRY(pool_alloc(reinterpret_cast<void**>(&ysq), sizeof(float) * rows_max));
  KNN_TRY(pool_alloc(reinterpret_cast<void**>(&yabs), 2 * sizeof(float)));
  KNN_TRY(pool_alloc(reinterpret_cast<void**>(&stats), sizeof(Stats)));
  KNN_TRY(pool_alloc(reinterpret_cast<void**>(&tab2orig), sizeof(uint32_t) * rows_max));
  KNN_TRY(pool_alloc(reinterpret_cast<void**>(&topk), sizeof(float) * static_cast<size_t>(kk) * stride));
  KNN_TRY(pool_alloc(reinterpret_cast<void**>(&dub), sizeof(float) * stride));
  KNN_TRY(pool_alloc(reinterpret_cast<void**>(&kcnt), sizeof(uint32_t) * stride));
  KNN_TRY(pool_alloc(reinterpret_cast<void**>(&kflags), sizeof(uint32_t) * stride));
  KNN_TRY(pool_alloc(reinterpret_cast<void**>(&entries), sizeof(uint4) * static_cast<size_t>(stride) * KNN_CAP));
  KNN_TRY(pool_alloc(reinterpret_cast<void**>(&ranges1), sizeof(uint2) * 2ull * tmax));
  KNN_TRY(pool_alloc(reinterpret_cast<void**>(&pool), sizeof(uint2) * pool_cap));
  KNN_TRY(pool_alloc(reinterpret_cast<void**>(&pair_row), sizeof(uint32_t) * pair_cap));
  KNN_TRY(pool_alloc(reinterpret_cast<void**>(&pair_cand), sizeof(uint32_t) * pair_cap));
  KNN_TRY(pool_alloc(reinterpret_cast<void**>(&pair_score), sizeof(float) * pair_cap));
  KNN_TRY(pool_alloc(reinterpret_cast<void**>(&rowq), sizeof(uint32_t) * 3ull * nv));
  KNN_TRY(pool_alloc(reinterpret_cast<void**>(&counters), sizeof(uint32_t) * CNT_N));
  KNN_TRY(cudaMemsetAsync(counters, 0, sizeof(uint32_t) * CNT_N, st));
  KNN_TRY(cudaMemsetAsync(stats, 0, sizeof(Stats), st));
  KNN_TRY(cudaMemsetAsync(yabs, 0, 2 * sizeof(float), st));
  KNN_TRY(cudaMemsetAsync(ysq, 0, sizeof(float) * rows_max, st));   // rows past the last block stay 0 for the max
  KNN_TRY(cudaMemsetAsync(kcnt, 0, sizeof(uint32_t) * stride, st));
  KNN_TRY(cudaMemsetAsync(kflags, 0, sizeof(uint32_t) * stride, st));
  KNN_TRY(cudaMemsetAsync(tab2orig, 0xff, sizeof(uint32_t) * rows_max, st));
  KNN_TRY(tc_set_smem_attr(static_cast<int>(smem_bytes), nkb));
  // cluster-aligned table layout: blocks per cluster, first block of every cluster, table row -> sample
  knn::tile_count_kernel<<<(K + 255) / 256, 256, 0, st>>>(off, K, ntile);
  KNN_TRY(cub::DeviceScan::ExclusiveSum(nullptr, cub_bytes, ntile, blk_first, static_cast<int>(K), st));
  KNN_TRY(pool_alloc(reinterpret_cast<void**>(&cub_tmp), cub_bytes ? cub_bytes : 16));
  KNN_TRY(cub::DeviceScan::ExclusiveSum(cub_tmp, cub_bytes, ntile, blk_first, static_cast<int>(K), st));
  knn::tile_fill_kernel<<<(K + 255) / 256, 256, 0, st>>>(off, K, blk_first, t_nrows, blk_cluster, ranges1, roff1, rcount1,
                                                         nblk1, d_ntiles, d_pairs);
  KNN_TRY(cudaMemcpyAsync(blk_first + K, d_ntiles, sizeof(uint32_t), cudaMemcpyDeviceToDevice, st));
  knn::layout_kernel<<<(nv + 255) / 256, 256, 0, st>>>(inv, assign, off, blk_first, nv, tab2orig);
  // fp16 table of the centred samples + bias blobs + statistics
  knn::prep_norms_kernel<<<(rows_max / 8) + 1, 256, 0, st>>>(X, C, D, tab2orig, blk_cluster, d_ntiles, ysq, yabs, metric);
  tc_prep_stats_kernel<<<8, 256, 0, st>>>(ysq, rows_max, stats);
  tc_prep_scale_kernel<<<1, 1, 0, st>>>(stats);
  knn::prep_table_kernel<<<(rows_max / 8) + 1, 256, 0, st>>>(X, C, D, nkb, tab2orig, blk_cluster, d_ntiles, ysq, table,
                                                             blobs, stats, yabs, metric, d_err);
  KNN_TRY(cudaGetLastError());
  KNN_TRY(encode_table_map(&tmap, table, rows_max, nkb));
  // (Params::metric stays 0: both metrics take the L2 candidate pass, the angular one on unit-length samples)
  prm.n = N; prm.D = D; prm.K = K; prm.nkb = nkb;
  prm.aug_blob = blobs; prm.stats = stats; prm.counters = counters;
  prm.X = X; prm.rows = tab2orig; prm.d_ntiles = d_ntiles; prm.tile_nrows = t_nrows;
  prm.blk_cluster = blk_cluster; prm.C = C;
  prm.knn_ranges = ranges1; prm.knn_roff = roff1; prm.knn_rcount = rcount1; prm.knn_nblk = nblk1;
  prm.kk = kk; prm.knn_first_pass = 1; prm.knn_stride = stride; prm.knn_topk = topk;
  prm.knn_cnt = kcnt; prm.knn_flags = kflags; prm.knn_dub = dub; prm.knn_entries = entries;
  prm.knn_part = part; prm.knn_nparts = nparts ? nparts : 1;
  tc_launch(2, false, nkb, grid, smem_bytes, st, tmap, prm);
  KNN_TRY(cudaGetLastError());
  (t64 ? knn::range_build_kernel<4> : knn::range_build_kernel<2>)<<<num_sms * 4, 256, 0, st>>>(d_ntiles, t_nrows, blk_cluster, blk_first, off, K, cd, radii, ysq,
                                                       dub, pool, pool_cap, pool_used, roff2, rcount2, nblk2, d_err,
                                                       d_pairs, part, prm.knn_nparts);
  KNN_TRY(cudaGetLastError());
  prm.knn_ranges = pool; prm.knn_roff = roff2; prm.knn_rcount = rcount2; prm.knn_nblk = nblk2; prm.knn_first_pass = 0;
  tc_launch(2, false, nkb, grid, smem_bytes, st, tmap, prm);
  KNN_TRY(cudaGetLastError());
  (t64 ? knn::expand_kernel<4> : knn::expand_kernel<2>)<<<num_sms * 8, 256, 0, st>>>(d_ntiles, kk, stride, topk, kcnt, kflags, entries, tab2orig, pair_cap,
                                                  pair_row, pair_cand, rowq, fb_rows, counters, pool_used + 2, part,
                                                  prm.knn_nparts);
  KNN_TRY(cudaGetLastError());
  // the exact distance of every candidate pair in the CALLER's metric (angular: acos of the Kahan dot product)
  launch_recheck_pairs<1>(metric, num_sms * 4, st, X, X, nullptr, D, pair_row, pair_cand, counters + CNT_PAIRS,
                          pair_cap, N, N, pair_score);
  knn::select_kernel<<<num_sms * 8, 256, 0, st>>>(k, rowq, counters, pair_cand, pair_score, 0u, neighbors);
  KNN_TRY(cudaGetLastError());
  KNN_TRY(cudaMemcpyAsync(h_cnt, counters, sizeof(uint32_t) * CNT_N, cudaMemcpyDeviceToHost, st));
  KNN_TRY(cudaMemcpyAsync(h_cnt + CNT_N, d_err, sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
  KNN_TRY(cudaMemcpyAsync(d_nfb, counters + CNT_OVF, sizeof(uint32_t), cudaMemcpyDeviceToDevice, st));
  KNN_TRY(cudaMemcpyAsync(h_dbg, pool_used + 2, sizeof(h_dbg), cudaMemcpyDeviceToHost, st));
  KNN_TRY(cudaStreamSynchronize(st));
  *h_error = h_cnt[CNT_ERR] | (h_cnt[CNT_N] ? 0x80000000u : 0u);
  if (getenv("KMCUDA_B200_TIMING"))
    fprintf(stderr, "[kmcuda_b200 timing]   knn tensor-core path: %u rows, %u candidate pairs, %u rows to the exact search, "
            "error word 0x%x; fallback reasons: nan/inf %u, list full %u, tiny diff %u, no threshold %u, >64 cand %u, "
            "<k cand %u; candidates seen %u\n", h_cnt[CNT_ROWQ], h_cnt[CNT_PAIRS], h_cnt[CNT_OVF], *h_error, h_dbg[0],
            h_dbg[1], h_dbg[2], h_dbg[3], h_dbg[4], h_dbg[5], h_dbg[6]);
done:
  pool_free(u32); pool_free(table); pool_free(blobs); pool_free(ysq); pool_free(yabs); pool_free(stats); pool_free(tab2orig);
  pool_free(topk); pool_free(dub); pool_free(kcnt); pool_free(kflags); pool_free(entries); pool_free(ranges1);
  pool_free(pool); pool_free(pair_row); pool_free(pair_cand); pool_free(pair_score); pool_free(rowq); pool_free(counters);
  pool_free(cub_tmp);
  return e;
}
#undef KNN_TRY

}  // namespace kmb
