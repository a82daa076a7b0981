// yinyang.cu -- one Yinyang iteration on a shard (reference kmeans_yy_global_filter + kmeans_yy_local_filter,
// kmeans.cu:540-672), restructured for the tensor-core filter:
//
//   * bounds are one contiguous [G+1] record per sample (the reference keeps [(G+1)][N] planes), so the group
//     filter is a single coalesced stream and a surviving sample's record is one 412-byte read (G = 102);
//   * the upper bound is tightened with the exact distance kernel over a compacted list (coalesced staging)
//     instead of a divergent per-thread loop inside the filter;
//   * the local filter's "scan all centroids of the unpruned groups" is replaced by the tensor-core (wgmma) candidate
//     pass (assign_tc.cu, MODE 1): only centroids whose fp16 score is within the rigorous margin of the
//     sample's second best are evaluated exactly.  The reference's outputs of that scan are the smallest and
//     second smallest element of the multiset {ub} U {exact distances of unpruned centroids} U {lower bounds
//     of pruned groups}; with valid bounds every element that can be among the two smallest is a candidate,
//     so (nearest, ub, lb[group(nearest)]) come out as in the reference (kmeans.cu:620-668).
//
// All bound arithmetic is the reference's fp32 sequence; distances are the exact kernels of exact.cuh.
#include <cfloat>
#include <cstdint>

#include "exact.cuh"
#include "kernels.h"

namespace kmb {

namespace {

enum { YC_TIGHT = 0, YC_PASSED = 1 };

__global__ void yy_group_sizes_kernel(const uint32_t* __restrict__ groups, uint32_t K, uint32_t G,
                                      uint32_t* __restrict__ gsize) {
  uint32_t c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c < K && groups[c] < G) atomicAdd(&gsize[groups[c]], 1u);
}

// warp-batched list append: lane `pending` keeps the row until 32 are collected
struct WarpAppender {
  uint32_t mine = 0, mine2 = 0;
  int pending = 0;
  __device__ void push(int lane, uint32_t row, uint32_t aux, uint32_t* counter, uint32_t* list, uint32_t* list2) {
    if (lane == pending) { mine = row; mine2 = aux; }
    pending++;
    if (pending == 32) flush(lane, counter, list, list2);
  }
  __device__ void flush(int lane, uint32_t* counter, uint32_t* list, uint32_t* list2) {
    if (pending == 0) return;
    uint32_t base = 0;
    if (lane == 0) base = atomicAdd(counter, static_cast<uint32_t>(pending));
    base = __shfl_sync(0xffffffffu, base, 0);
    if (lane < pending) {
      list[base + lane] = mine;
      if (list2) list2[base + lane] = mine2;
    }
    pending = 0;
  }
};

// kmeans.cu:548-570: ub += drift[a]; lb[g] -= maxdrift[g]; rows with min lb >= ub are done
__global__ void __launch_bounds__(256)
yy_decay_kernel(uint32_t n, uint32_t K, uint32_t G, const float* __restrict__ drift, const float* __restrict__ maxdrift,
                const uint32_t* __restrict__ assign, uint32_t* __restrict__ prev, float* __restrict__ bounds,
                float* __restrict__ minlb_out, uint32_t* __restrict__ tight_rows, uint32_t* __restrict__ tight_cand,
                uint32_t* __restrict__ counters) {
  const int lane = threadIdx.x & 31;
  const uint32_t warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, nwarps = (gridDim.x * blockDim.x) >> 5;
  WarpAppender app;
  for (uint32_t row = warp; row < n; row += nwarps) {
    float* b = bounds + static_cast<size_t>(row) * (G + 1);
    const uint32_t a = assign[row];
    if (a >= K) {   // "insane" sample (first feature NaN): never reassigned
      if (lane == 0) prev[row] = a;
      continue;
    }
    const float ub = b[0] + drift[a];
    float mn = FLT_MAX;
    for (uint32_t g = lane; g < G; g += 32) {
      const float lb = b[1 + g] - __ldg(maxdrift + g);
      b[1 + g] = lb;
      if (lb < mn) mn = lb;
    }
    for (int o = 16; o > 0; o >>= 1) mn = fminf(mn, __shfl_xor_sync(0xffffffffu, mn, o));
    if (lane == 0) prev[row] = a;
    if (mn >= ub) {
      if (lane == 0) b[0] = ub;
    } else {
      if (lane == 0) minlb_out[row] = mn;
      app.push(lane, row, a, &counters[YC_TIGHT], tight_rows, tight_cand);
    }
  }
  app.flush(lane, &counters[YC_TIGHT], tight_rows, tight_cand);
}

// kmeans.cu:571-580: ub = exact distance to the own centroid; rows with min lb < ub go to the local step
__global__ void yy_pass_kernel(uint32_t G, const uint32_t* __restrict__ tight_rows,
                               const float* __restrict__ tight_score, const float* __restrict__ minlb,
                               float* __restrict__ bounds, uint32_t* __restrict__ passed,
                               uint32_t* __restrict__ counters) {
  const uint32_t nt = counters[YC_TIGHT];
  const int lane = threadIdx.x & 31;
  for (uint32_t i0 = (blockIdx.x * blockDim.x + threadIdx.x) & ~31u; i0 < nt; i0 += gridDim.x * blockDim.x) {
    const uint32_t i = i0 + lane;
    bool pass = false;
    uint32_t row = 0;
    if (i < nt) {
      row = tight_rows[i];
      const float ub = tight_score[i];
      bounds[static_cast<size_t>(row) * (G + 1)] = ub;
      pass = !(minlb[row] >= ub);
    }
    const unsigned m = __ballot_sync(0xffffffffu, pass);
    if (m) {
      uint32_t base = 0;
      if (lane == 0) base = atomicAdd(&counters[YC_PASSED], static_cast<uint32_t>(__popc(m)));
      base = __shfl_sync(0xffffffffu, base, 0);
      if (pass) passed[base + __popc(m & ((1u << lane) - 1))] = row;
    }
  }
}

// One warp per surviving row: merge the exact candidate distances with the pruned groups' lower bounds
// (kmeans.cu:620-668).  mn / nearest = smallest element (the own centroid wins ties, then the lowest index),
// sec = second smallest element of the multiset.
__global__ void __launch_bounds__(256)
yy_finish_kernel(uint32_t G, const uint32_t* __restrict__ groups, const uint32_t* __restrict__ gsize,
                 const uint32_t* __restrict__ rowq, const uint32_t* __restrict__ d_nrowq,
                 const uint32_t* __restrict__ pair_cand, const float* __restrict__ pair_score,
                 uint32_t* __restrict__ assign, float* __restrict__ bounds, uint32_t* __restrict__ d_changed) {
  const uint32_t nq = *d_nrowq;
  const int lane = threadIdx.x & 31;
  const uint32_t warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, nwarps = (gridDim.x * blockDim.x) >> 5;
  uint32_t changed = 0;
  for (uint32_t q = warp; q < nq; q += nwarps) {
    const uint32_t row = rowq[3 * q], base = rowq[3 * q + 1], cnt = rowq[3 * q + 2];
    if (cnt == 0) continue;   // neutralised slot: the row is on the overflow list
    float* b = bounds + static_cast<size_t>(row) * (G + 1);
    const float ub = b[0];
    const uint32_t a = assign[row];
    const uint32_t pg = groups[a];
    // pruned groups contribute their lower bound; every such bound is >= ub >= the minimum, so only the
    // smallest one can be the second smallest element
    float p1 = FLT_MAX;
    for (uint32_t g = lane; g < G; g += 32) {
      const float lb = b[1 + g];
      if (!(lb >= ub)) continue;
      if (gsize[g] - (g == pg ? 1u : 0u) == 0) continue;   // no member besides the own centroid: never visited
      if (lb < p1) p1 = lb;
    }
    // this lane's candidate (exact distance), dropped if it is the own centroid or sits in a pruned group
    float d = FLT_MAX;
    uint32_t c = UINT32_MAX;
    if (static_cast<uint32_t>(lane) < cnt) {
      const uint32_t cc = pair_cand[base + lane];
      const uint32_t g = groups[cc];
      const float dd = pair_score[base + lane];
      if (cc != a && g < G && !(b[1 + g] >= ub) && dd == dd) { d = dd; c = cc; }
    }
    // warp-wide two smallest over {candidates} and {pruned bounds}
    float dmin = d;
    for (int o = 16; o > 0; o >>= 1) dmin = fminf(dmin, __shfl_xor_sync(0xffffffffu, dmin, o));
    uint32_t cbest = (c != UINT32_MAX && d == dmin) ? c : UINT32_MAX;
    for (int o = 16; o > 0; o >>= 1) cbest = min(cbest, __shfl_xor_sync(0xffffffffu, cbest, o));
    const bool moved = cbest != UINT32_MAX && dmin < ub;          // strict '<' from mn = ub (kmeans.cu:652)
    const uint32_t near = moved ? cbest : a;
    const float mn = moved ? dmin : ub;
    // second smallest: drop ONE instance of the minimum (the lane holding `near`), then take the minimum of the rest
    float rest = (moved && c == cbest) ? FLT_MAX : d;              // candidate indices are unique per row
    rest = fminf(rest, p1);
    for (int o = 16; o > 0; o >>= 1) rest = fminf(rest, __shfl_xor_sync(0xffffffffu, rest, o));
    float sec = moved ? fminf(ub, rest) : rest;
    if (lane == 0) {
      const uint32_t ng = groups[near];
      if (ng < G) b[1 + ng] = sec;
      if (ng != pg && pg < G) {
        if (b[1 + pg] > ub) b[1 + pg] = ub;
      }
      b[0] = mn;
      if (near != a) {
        assign[row] = near;
        changed++;
      }
    }
  }
  if (lane == 0 && changed) atomicAdd(d_changed, changed);
}

// Reference-order scan for the rows the tensor-core pass could not bound (and for shapes it does not
// support): kmeans.cu:584-672 restated with row-major samples, one thread per listed row.
template <int METRIC>
__global__ void yy_local_scan_kernel(const float* __restrict__ X, const float* __restrict__ C, int D, uint32_t K,
                                     uint32_t G, const uint32_t* __restrict__ groups,
                                     const float* __restrict__ drift, const float* __restrict__ maxdrift,
                                     const uint32_t* __restrict__ rows, const uint32_t* __restrict__ d_nrows,
                                     uint32_t* __restrict__ assign, float* __restrict__ bounds,
                                     uint32_t* __restrict__ d_changed) {
  const uint32_t np = *d_nrows;
  int changed = 0;
  for (uint32_t p = blockIdx.x * blockDim.x + threadIdx.x; p < np; p += gridDim.x * blockDim.x) {
    const uint32_t i = rows[p];
    float* b = bounds + static_cast<size_t>(i) * (G + 1);
    const float ub = b[0];
    const uint32_t a = assign[i];
    float mn = ub, sec = FLT_MAX;
    uint32_t near = a;
    const float* x = X + static_cast<size_t>(i) * D;
    for (uint32_t c = 0; c < K; c++) {
      if (c == a) continue;
      const uint32_t g = groups[c];
      if (g >= G) continue;
      float lb = b[1 + g];
      if (lb >= ub) {
        if (lb < sec) sec = lb;
        continue;
      }
      lb += maxdrift[g] - drift[c];
      if (sec < lb) continue;
      const float d = distance_exact<METRIC>(x, C + static_cast<size_t>(c) * D, D);
      if (d < mn) {
        sec = mn;
        mn = d;
        near = c;
      } else if (d < sec) {
        sec = d;
      }
    }
    const uint32_t ng = groups[near], pg = groups[a];
    if (ng < G) b[1 + ng] = sec;
    if (ng != pg && pg < G) {
      if (b[1 + pg] > ub) b[1 + pg] = ub;
    }
    b[0] = mn;
    if (near != a) {
      assign[i] = near;
      changed++;
    }
  }
  for (int o = 16; o > 0; o >>= 1) changed += __shfl_down_sync(0xffffffffu, changed, o);
  if ((threadIdx.x & 31) == 0 && changed) atomicAdd(d_changed, changed);
}

// One CTA per listed row: exact distances to every centroid of the unpruned groups, spread over the 256 threads
// (rows the tensor-core pass could not bound, and every surviving row of shapes it does not support).  Same
// result as the scan above whenever the bounds are valid: the scan's second-level skip (kmeans.cu:644-646) only
// omits centroids that cannot be among the two smallest.
template <int METRIC>
__global__ void __launch_bounds__(256)
yy_rows_cta_kernel(const float* __restrict__ X, const float* __restrict__ C, int D, uint32_t K, uint32_t G,
                   const uint32_t* __restrict__ groups, const uint32_t* __restrict__ rows,
                   const uint32_t* __restrict__ d_nrows, uint32_t* __restrict__ assign, float* __restrict__ bounds,
                   uint32_t* __restrict__ d_changed, int smem_d) {
  extern __shared__ float sx[];   // [smem_d]: the row (smem_d == D), or nothing (smem_d == 0: read X directly)
  __shared__ float s_d1[256], s_d2[256], s_p[256];
  __shared__ uint32_t s_c1[256];
  const uint32_t nrows = *d_nrows;
  const int tid = threadIdx.x;
  for (uint32_t e = blockIdx.x; e < nrows; e += gridDim.x) {
    const uint32_t row = rows[e];
    float* b = bounds + static_cast<size_t>(row) * (G + 1);
    const float* xs = X + static_cast<size_t>(row) * D;
    __syncthreads();
    if (smem_d) {
      for (int f = tid; f < D; f += 256) sx[f] = xs[f];
      xs = sx;
    }
    const float ub = b[0];
    const uint32_t a = assign[row];
    __syncthreads();
    float d1 = FLT_MAX, d2 = FLT_MAX, pl = FLT_MAX;
    uint32_t c1 = UINT32_MAX;
    // four independent Kahan chains per thread (centroids tid, tid+256, ...) hide the dependent-add latency
    for (uint32_t c0 = tid; c0 < K; c0 += 1024) {
      const float* cp[4];
      bool live[4];
#pragma unroll
      for (int j = 0; j < 4; j++) {
        const uint32_t c = c0 + 256u * j;
        live[j] = false;
        cp[j] = C;
        if (c < K && c != a) {
          const uint32_t g = groups[c];
          if (g < G) {
            const float lb = b[1 + g];
            if (lb >= ub) {
              if (lb < pl) pl = lb;
            } else {
              live[j] = true;
              cp[j] = C + static_cast<size_t>(c) * D;
            }
          }
        }
      }
      if (!(live[0] || live[1] || live[2] || live[3])) continue;
      Kahan k[4];
      for (int f = 0; f < D; f++) {
        const float x = xs[f];
#pragma unroll
        for (int j = 0; j < 4; j++) {
          const float cv = __ldg(cp[j] + f);
          if (METRIC == 1) k[j].mac(x, cv);
          else k[j].sqdiff(x, cv);
        }
      }
#pragma unroll
      for (int j = 0; j < 4; j++) {   // ascending centroid index within the thread: strict '<' keeps the lowest
        if (!live[j]) continue;
        const float d = finalize_distance<METRIC>(k[j].sum);
        if (d < d1) {
          d2 = d1;
          d1 = d;
          c1 = c0 + 256u * j;
        } else if (d < d2) {
          d2 = d;
        }
      }
    }
    s_d1[tid] = d1; s_d2[tid] = d2; s_p[tid] = pl; s_c1[tid] = c1;
    __syncthreads();
    for (int o = 128; o > 0; o >>= 1) {
      if (tid < o) {
        const float a1 = s_d1[tid], b1 = s_d1[tid + o];
        const uint32_t ac = s_c1[tid], bc = s_c1[tid + o];
        const float second = fminf(fmaxf(a1, b1), fminf(s_d2[tid], s_d2[tid + o]));
        if (b1 < a1 || (b1 == a1 && bc < ac)) {
          s_d1[tid] = b1;
          s_c1[tid] = bc;
        }
        s_d2[tid] = second;
        s_p[tid] = fminf(s_p[tid], s_p[tid + o]);
      }
      __syncthreads();
    }
    if (tid == 0) {
      d1 = s_d1[0]; d2 = s_d2[0]; pl = s_p[0]; c1 = s_c1[0];
      const bool moved = c1 != UINT32_MAX && d1 < ub;
      const uint32_t near = moved ? c1 : a;
      const float mn = moved ? d1 : ub;
      const float sec = moved ? fminf(ub, fminf(d2, pl)) : fminf(d1, pl);
      const uint32_t ng = groups[near], pg = groups[a];
      if (ng < G) b[1 + ng] = sec;
      if (ng != pg && pg < G) {
        if (b[1 + pg] > ub) b[1 + pg] = ub;
      }
      b[0] = mn;
      if (near != a) {
        assign[row] = near;
        atomicAdd(d_changed, 1u);
      }
    }
  }
}

// exact distance to the own centroid for listed rows when no tensor-core plan exists (thread per row)
template <int METRIC>
__global__ void yy_tight_scan_kernel(const float* __restrict__ X, const float* __restrict__ C, int D,
                                     const uint32_t* __restrict__ rows, const uint32_t* __restrict__ cand,
                                     const uint32_t* __restrict__ d_n, float* __restrict__ out) {
  const uint32_t nt = *d_n;
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < nt; i += gridDim.x * blockDim.x)
    out[i] = distance_exact<METRIC>(X + static_cast<size_t>(rows[i]) * D, C + static_cast<size_t>(cand[i]) * D, D);
}

}  // namespace

cudaError_t launch_yy_group_sizes(const uint32_t* groups, uint32_t K, uint32_t G, uint32_t* gsize, cudaStream_t st) {
  cudaError_t e = cudaMemsetAsync(gsize, 0, sizeof(uint32_t) * G, st);
  if (e != cudaSuccess) return e;
  yy_group_sizes_kernel<<<(K + 255) / 256, 256, 0, st>>>(groups, K, G, gsize);
  return cudaGetLastError();
}

cudaError_t launch_yy_step(int metric, TcPlan* plan, const float* X, const float* C, const float* csq, uint32_t n,
                           int D, uint32_t K, uint32_t G, const uint32_t* groups, const float* drift,
                           const float* maxdrift, uint32_t* assign, uint32_t* prev, float* bounds,
                           const YyWorkspace& ws, uint32_t* d_changed, bool reference_order_scan, cudaStream_t st) {
  if (n == 0) return cudaSuccess;
  cudaError_t e;
  if ((e = cudaMemsetAsync(ws.counters, 0, sizeof(uint32_t) * 4, st)) != cudaSuccess) return e;
  const unsigned sgrid = device_sms() * 8;
  yy_decay_kernel<<<sgrid, 256, 0, st>>>(n, K, G, drift, maxdrift, assign, prev, bounds, ws.minlb,
                                                        ws.tight_rows, ws.tight_cand, ws.counters);
  if ((e = cudaGetLastError()) != cudaSuccess) return e;
  if (plan) {
    if ((e = tc_exact_distances(plan, X, C, n, ws.tight_rows, ws.tight_cand, ws.counters + YC_TIGHT, n,
                                ws.tight_score, st)) != cudaSuccess)
      return e;
  } else {
    if (metric == 1)
      yy_tight_scan_kernel<1><<<sgrid, 128, 0, st>>>(X, C, D, ws.tight_rows, ws.tight_cand, ws.counters + YC_TIGHT,
                                                     ws.tight_score);
    else
      yy_tight_scan_kernel<0><<<sgrid, 128, 0, st>>>(X, C, D, ws.tight_rows, ws.tight_cand, ws.counters + YC_TIGHT,
                                                     ws.tight_score);
  }
  yy_pass_kernel<<<sgrid, 256, 0, st>>>(G, ws.tight_rows, ws.tight_score, ws.minlb, bounds, ws.passed, ws.counters);
  if ((e = cudaGetLastError()) != cudaSuccess) return e;
  const uint32_t* scan_rows = ws.passed;
  const uint32_t* scan_n = ws.counters + YC_PASSED;
  if (plan) {
    if ((e = tc_yy_candidates(plan, X, C, csq, n, ws.passed, ws.counters + YC_PASSED, st)) != cudaSuccess) return e;
    TcQueues q;
    tc_queues(plan, &q);
    yy_finish_kernel<<<sgrid, 256, 0, st>>>(G, groups, ws.gsize, q.rowq, q.d_nrowq, q.pair_cand, q.pair_score, assign,
                                           bounds, d_changed);
    if ((e = cudaGetLastError()) != cudaSuccess) return e;
    scan_rows = q.ovf_rows;
    scan_n = q.d_novf;
  }
  if (reference_order_scan) {
    if (metric == 1)
      yy_local_scan_kernel<1><<<sgrid, 128, 0, st>>>(X, C, D, K, G, groups, drift, maxdrift, scan_rows, scan_n, assign,
                                                     bounds, d_changed);
    else
      yy_local_scan_kernel<0><<<sgrid, 128, 0, st>>>(X, C, D, K, G, groups, drift, maxdrift, scan_rows, scan_n, assign,
                                                     bounds, d_changed);
  } else {
    const int smem_d = D <= kRowStageMaxD ? D : 0;
    const size_t smem = sizeof(float) * smem_d;
    auto kern = metric == 1 ? yy_rows_cta_kernel<1> : yy_rows_cta_kernel<0>;
    if ((e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem))) !=
        cudaSuccess)
      return e;
    kern<<<device_sms() * 8, 256, smem, st>>>(X, C, D, K, G, groups, scan_rows, scan_n, assign, bounds, d_changed,
                                              smem_d);
  }
  return cudaGetLastError();
}

}  // namespace kmb
