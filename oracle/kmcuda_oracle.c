/*
 * kmcuda_oracle.c -- TEST INFRASTRUCTURE ONLY (never linked into, called by, or shipped with the
 * product library).  Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline /
 * --impl reference legs may load this file's shared object.
 *
 * CPU restatement of the arithmetic of src-d/kmcuda's batched-distance hot path, written from the
 * reference's *behaviour* (file:line citations are to /root/reference/src).  fp32 path only; the
 * reference's fp16x2 path accumulates in fp16 and has no bit-wise parity contract (SURVEY.md 7.2).
 *
 * Parity pin: on the GPU box this restatement is compared bit-for-bit against the UNMODIFIED
 * reference rebuilt for sm_90 (oracle/_ref/libKMCUDA.so, see oracle/build_ref.sh) by
 * tests/test_parity_gpu.py::test_oracle_matches_reference_*; on the CPU it is pinned against
 * scikit-learn the same way the reference's own test.py pins the reference (tests/test_oracle_cpu.py).
 * Cosine uses the host libm acosf, which is NOT bit-specified to equal CUDA's acosf: cosine results
 * are exact only up to acos rounding ties (documented in DESIGN.md).
 *
 * Arithmetic spec (SURVEY.md Appendix A):
 *   fma_rd(a,b,c) = a*b+c rounded toward -inf              fp_abstraction.h:88-90 (__fmaf_rd)
 *   all other +,- are round-to-nearest fp32                 fp_abstraction.h:72-82
 *   reciprocal = correctly rounded 1/x                      fp_abstraction.h:84-86 (__frcp_rn)
 *   sqrt = correctly rounded                                fp_abstraction.h:96-98 (__fsqrt_rn)
 */
#include <math.h>
#include <float.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>
#include <stdio.h>

#ifdef _OPENMP
#include <omp.h>
#endif

/* launchers such as torchrun export OMP_NUM_THREADS=1; the timing legs set the thread count explicitly */
int ko_set_threads(int n) {
#ifdef _OPENMP
  if (n > 0) omp_set_num_threads(n);
  return omp_get_max_threads();
#else
  (void)n;
  return 1;
#endif
}

#define KO_L2 0
#define KO_COS 1

/* ------------------------------------------------------------------------------------------ */
/* round-toward-minus-infinity fused multiply-add without touching the FP environment.         */
/* a*b is exact in double (24x24 bits); TwoSum gives the exact error of the double addition,   */
/* so the exact value s+e is known and RN-to-float can be corrected downwards.                 */
/* ------------------------------------------------------------------------------------------ */
float ko_fma_rd(float a, float b, float c) {
  double p = (double)a * (double)b;
  double cd = (double)c;
  double s = p + cd;
  if (!(s == s) || isinf(s)) return (float)s;
  double bb = s - p;
  double e = (p - (s - bb)) + (cd - bb);
  if (s == 0.0 && e == 0.0) {
    /* exact zero: round-down yields -0 unless both addends are +0 */
    if (p == 0.0 && cd == 0.0 && !signbit(p) && !signbit(cd)) return 0.0f;
    return -0.0f;
  }
  float f = (float)s;
  double fd = (double)f;
  if (fd > s || (fd == s && e < 0.0)) f = nextafterf(f, -INFINITY);
  return f;
}

/* Kahan dot product "with inverted c": kmeans.cu:331-341, metric_abstraction.h:182-193 */
float ko_kahan_dot(const float *a, const float *b, int D) {
  float p = 0.f, r = 0.f;
  for (int f = 0; f < D; f++) {
    float y = ko_fma_rd(a[f], b[f], r);
    float t = p + y;
    r = y - (t - p);
    p = t;
  }
  return p;
}

/* squared norm: metric_abstraction.h:21-36 (L2); cosine returns the constant 1 (:149-158) */
float ko_csqr(int metric, const float *c, int D) {
  if (metric == KO_COS) return 1.f;
  float q = 0.f, r = 0.f;
  for (int f = 0; f < D; f++) {
    float y = ko_fma_rd(c[f], c[f], r);
    float t = q + y;
    r = y - (t - q);
    q = t;
  }
  return q;
}

/* Kahan sum of squared differences: metric_abstraction.h:59-71, 73-86, 88-101 */
static float ko_sqdiff(const float *a, const float *b, int D) {
  float q = 0.f, r = 0.f;
  for (int f = 0; f < D; f++) {
    float d = a[f] - b[f];
    float y = ko_fma_rd(d, d, r);
    float t = q + y;
    r = y - (t - q);
    q = t;
  }
  return q;
}

static float ko_acos_clamped(float p) { /* metric_abstraction.h:171-177, 250-254 */
  if (p >= 1.f) return 0.f;
  if (p <= -1.f) return (float)M_PI;
  return acosf(p);
}

/* ranking score used by the Lloyd assignment: metric_abstraction.h:55-57 (L2), :171-177 (cos) */
float ko_lloyd_score(int metric, const float *s, const float *c, float csqr, int D) {
  float prod = ko_kahan_dot(s, c, D);
  if (metric == KO_COS) return ko_acos_clamped(prod);
  return ko_fma_rd(-2.f, prod, 0.f + csqr);
}

/* true distance used by Yinyang / k-NN / average distance: metric_abstraction.h:59-101, 179-222 */
float ko_distance(int metric, const float *a, const float *b, int D) {
  if (metric == KO_COS) return ko_acos_clamped(ko_kahan_dot(a, b, D));
  return sqrtf(ko_sqdiff(a, b, D));
}

/* ------------------------------------------------------------------------------------------ */
/* Lloyd assignment pass: kmeans.cu:293-364.  Strict '<' in ascending centroid order; a sample  */
/* whose first feature is NaN is "insane" and gets K; if no centroid wins the assignment is     */
/* left untouched.  Returns the number of changed assignments (d_changed_number).               */
/* best_out/second_out (optional) receive the winning and runner-up fp32 scores.                */
/* ------------------------------------------------------------------------------------------ */
uint32_t ko_assign_lloyd(int metric, const float *X, const float *C, uint32_t N, int D, uint32_t K,
                         uint32_t *assign, uint32_t *prev, float *best_out, float *second_out) {
  float *csq = (float *)malloc(sizeof(float) * K);
  for (uint32_t c = 0; c < K; c++) csq[c] = ko_csqr(metric, C + (size_t)c * D, D);
  uint32_t changed = 0;
#pragma omp parallel for schedule(static) reduction(+ : changed)
  for (uint32_t i = 0; i < N; i++) {
    const float *s = X + (size_t)i * D;
    uint32_t nearest = UINT32_MAX;
    float best = FLT_MAX, second = FLT_MAX;
    int insane = (s[0] != s[0]);
    if (!insane) {
      for (uint32_t c = 0; c < K; c++) {
        float d = ko_lloyd_score(metric, s, C + (size_t)c * D, csq[c], D);
        if (d < best) {
          second = best;
          best = d;
          nearest = c;
        } else if (d < second) {
          second = d;
        }
      }
    }
    if (best_out) best_out[i] = best;
    if (second_out) second_out[i] = second;
    if (nearest == UINT32_MAX) {
      if (!insane) continue; /* kmeans.cu:349-353: printf + return, nothing written */
      nearest = K;
    }
    uint32_t a = assign[i];
    if (prev) prev[i] = a;
    if (a != nearest) {
      assign[i] = nearest;
      changed++;
    }
  }
  free(csq);
  return changed;
}

/* float64 "truth": best / second-best squared-L2 (or angle) and argmin, used as the tie detector */
void ko_assign_truth(int metric, const float *X, const float *C, uint32_t N, int D, uint32_t K,
                     uint32_t *arg, double *best_out, double *second_out) {
  double *csq = (double *)malloc(sizeof(double) * K);
  for (uint32_t c = 0; c < K; c++) {
    double q = 0;
    for (int f = 0; f < D; f++) q += (double)C[(size_t)c * D + f] * (double)C[(size_t)c * D + f];
    csq[c] = q;
  }
#pragma omp parallel for schedule(static)
  for (uint32_t i = 0; i < N; i++) {
    const float *s = X + (size_t)i * D;
    double best = INFINITY, second = INFINITY;
    uint32_t a = UINT32_MAX;
    for (uint32_t c = 0; c < K; c++) {
      const float *cc = C + (size_t)c * D;
      double dot = 0;
      for (int f = 0; f < D; f++) dot += (double)s[f] * (double)cc[f];
      double d;
      if (metric == KO_COS) d = dot >= 1 ? 0 : (dot <= -1 ? M_PI : acos(dot));
      else d = csq[c] - 2 * dot;
      if (d < best) { second = best; best = d; a = c; }
      else if (d < second) second = d;
    }
    arg[i] = a; best_out[i] = best; second_out[i] = second;
  }
  free(csq);
}

/* ------------------------------------------------------------------------------------------ */
/* Centroid update: kmeans_adjust, kmeans.cu:366-429 + normalize, metric_abstraction.h:138-144, */
/* 255-272.  Incremental: C*=count, then +/- the samples that entered/left in sample order with */
/* ONE Kahan compensation scalar shared by all features and samples; then normalise.            */
/* ------------------------------------------------------------------------------------------ */
void ko_adjust(int metric, const float *X, uint32_t N, int D, uint32_t K, const uint32_t *prev,
               const uint32_t *cur, float *C, uint32_t *ccounts) {
#pragma omp parallel for schedule(dynamic, 8)
  for (uint32_t c = 0; c < K; c++) {
    float *cc = C + (size_t)c * D;
    uint32_t cnt = ccounts[c];
    float fc = (float)cnt;
    for (int f = 0; f < D; f++) cc[f] = cc[f] * fc;
    float corr = 0.f;
    for (uint32_t i = 0; i < N; i++) {
      uint32_t ta = cur[i], pa = prev[i];
      int sign = 0;
      if (pa == c && ta != c) { sign = -1; cnt--; }
      else if (pa != c && ta == c) { sign = 1; cnt++; }
      if (!sign) continue;
      const float *s = X + (size_t)i * D;
      float fs = (float)sign;
      for (int f = 0; f < D; f++) {
        float y = ko_fma_rd(s[f], fs, corr);
        float t = cc[f] + y;
        corr = y - (t - cc[f]);
        cc[f] = t;
      }
    }
    if (metric == KO_COS) {
      float norm = 0.f, r = 0.f;
      for (int f = 0; f < D; f++) {
        float v = cc[f];
        float y = ko_fma_rd(v, v, r);
        float t = norm + y;
        r = y - (t - norm);
        norm = t;
      }
      norm = 1.0f / sqrtf(norm);
      for (int f = 0; f < D; f++) cc[f] = cc[f] * norm;
    } else {
      float rc = 1.0f / (float)cnt; /* cnt==0 -> inf -> NaN centroid, by design kmeans.cu:425-427 */
      for (int f = 0; f < D; f++) cc[f] = cc[f] * rc;
    }
    ccounts[c] = cnt;
  }
}

/* mean distance to the own centroid: kmeans.cu:674-691, 1265-1300 (double accumulation) */
float ko_average_distance(int metric, const float *X, const float *C, uint32_t N, int D,
                          const uint32_t *assign) {
  double sum = 0;
  for (uint32_t i = 0; i < N; i++)
    sum += ko_distance(metric, X + (size_t)i * D, C + (size_t)assign[i] * D, D);
  return (float)(sum / N);
}

/* ------------------------------------------------------------------------------------------ */
/* k-means++ seeding on the host RNG: kmcuda.cc:262-333 with kernel kmeans.cu:42-67.            */
/* Uses the C library rand() exactly as the reference does (srand(seed) by the caller).         */
/* ------------------------------------------------------------------------------------------ */
void ko_init_plusplus(int metric, const float *X, uint32_t N, int D, uint32_t K, float *C) {
  float *dists = (float *)malloc(sizeof(float) * N);
  uint32_t first;
  do { first = (uint32_t)rand() % N; } while (X[(size_t)first * D] != X[(size_t)first * D]);
  memcpy(C, X + (size_t)first * D, sizeof(float) * D);
  for (uint32_t i = 1; i < K; i++) {
    double dist_sum = 0;
    const float *last = C + (size_t)(i - 1) * D;
    for (uint32_t s = 0; s < N; s++) {
      float d = 0;
      const float *x = X + (size_t)s * D;
      if (x[0] == x[0]) d = ko_distance(metric, x, last, D);
      if (i == 1 || d < dists[s]) dists[s] = d; else d = dists[s];
      dist_sum += d;
    }
    double choice = ((rand() + .0) / RAND_MAX);
    uint32_t choice_approx = (uint32_t)(choice * N);
    double choice_sum = choice * dist_sum;
    uint32_t j;
    if (choice_approx < 100) {
      double s2 = 0;
      for (j = 0; j < N && s2 < choice_sum; j++) s2 += dists[j];
    } else {
      double s2 = 0;
      for (uint32_t t = 0; t < choice_approx; t++) s2 += dists[t];
      if (s2 < choice_sum) {
        for (j = choice_approx; j < N && s2 < choice_sum; j++) s2 += dists[j];
      } else {
        for (j = choice_approx; j > 1 && s2 >= choice_sum; j--) s2 -= dists[j];
        j++;
      }
    }
    if (j == 0) j = 1;
    if (j > N) j = N;
    memcpy(C + (size_t)i * D, X + (size_t)(j - 1) * D, sizeof(float) * D);
  }
  free(dists);
}

/* Lloyd loop: kmeans.cu:934-1026.  Returns the iteration count; log==1 prints the contract line. */
static int ko_lloyd_loop(int metric, float tolerance, const float *X, uint32_t N, int D, uint32_t K,
                         float *C, uint32_t *ccounts, uint32_t *prev, uint32_t *assign, int log,
                         uint32_t *last_changed, int max_iter) {
  memset(ccounts, 0, sizeof(uint32_t) * K);
  memset(assign, 0xff, sizeof(uint32_t) * N);
  memset(prev, 0xff, sizeof(uint32_t) * N);
  for (int iter = 1;; iter++) {
    uint32_t changed = ko_assign_lloyd(metric, X, C, N, D, K, assign, prev, NULL, NULL);
    if (last_changed) *last_changed = changed;
    if (log) printf("iteration %d: %u reassignments\n", iter, changed);
    if ((float)changed <= tolerance * (float)N) return iter; /* kmeans.cu:707 float compare */
    if (max_iter > 0 && iter >= max_iter) return iter;
    ko_adjust(metric, X, N, D, K, prev, assign, C, ccounts);
  }
}

/* ------------------------------------------------------------------------------------------ */
/* The three pieces of a Yinyang iteration, on the reference's bound planes: bounds[g * N + i], */
/* plane 0 the upper bound, plane 1 + g the lower bound of group g.  ko_kmeans below calls      */
/* them, so the whole-run oracle and the single-step oracle are the same code.                  */
/* ------------------------------------------------------------------------------------------ */

/* bounds refresh: kmeans_yy_init, kmeans.cu:431-485 */
void ko_yy_init(int metric, const float *X, const float *C, uint32_t N, int D, uint32_t K, uint32_t G,
                const uint32_t *groups, const uint32_t *assign, float *bounds) {
#pragma omp parallel for schedule(static)
  for (uint32_t i = 0; i < N; i++) {
    for (uint32_t g = 0; g <= G; g++) bounds[(size_t)N * g + i] = FLT_MAX;
    uint32_t nearest = assign[i];
    for (uint32_t c = 0; c < K; c++) {
      uint32_t g = groups[c];
      if (g >= G) continue;
      float d = ko_distance(metric, X + (size_t)i * D, C + (size_t)c * D, D);
      if (c != nearest) {
        if (d < bounds[(size_t)N * (1 + g) + i]) bounds[(size_t)N * (1 + g) + i] = d;
      } else {
        bounds[i] = d;
      }
    }
  }
}

/* drifts, kmeans_yy_calc_drifts, kmeans.cu:487-499, and the group maxima,
 * kmeans_yy_find_group_max_drifts, kmeans.cu:501-538 (a group without members keeps -FLT_MAX) */
void ko_yy_drifts(int metric, const float *C, const float *oldC, uint32_t K, int D, uint32_t G,
                  const uint32_t *groups, float *drift, float *maxdrift) {
  for (uint32_t c = 0; c < K; c++)
    drift[c] = ko_distance(metric, C + (size_t)c * D, oldC + (size_t)c * D, D);
  for (uint32_t g = 0; g < G; g++) {
    float m = -FLT_MAX;
    for (uint32_t c = 0; c < K; c++) if (groups[c] == g && m < drift[c]) m = drift[c];
    maxdrift[g] = m;
  }
}

/* Global filter, kmeans.cu:540-582, then local filter, kmeans.cu:584-672.  Returns the number of
 * changed assignments; *tight_out = rows whose decayed lower bounds do not prune them (filter #1
 * fails, the upper bound is recomputed), *passed_out = rows that also fail filter #2 (local step).
 * Two guards are not in the reference, which reads or writes out of range there; both restate
 * the library's own (yinyang.cu):
 *   - a row assigned >= K ("insane", first feature NaN) gets prev = assign and keeps its bounds
 *     (the reference reads drift[K]);
 *   - no bound is written for a group >= G (the reference writes plane 1 + G, past the end). */
uint32_t ko_yy_step(int metric, const float *X, const float *C, uint32_t N, int D, uint32_t K, uint32_t G,
                    const uint32_t *groups, const float *drift, const float *maxdrift, uint32_t *assign,
                    uint32_t *prev, float *bounds, uint32_t *tight_out, uint32_t *passed_out) {
  uint32_t *passed = (uint32_t *)malloc(sizeof(uint32_t) * (N ? N : 1));
  uint32_t npassed = 0, ntight = 0;
  for (uint32_t i = 0; i < N; i++) {
    uint32_t a = assign[i];
    prev[i] = a;
    if (a >= K) continue; /* deviation: the library's guard (yy_decay_kernel) */
    float ub = bounds[i] + drift[a];
    float minlb = FLT_MAX;
    for (uint32_t g = 0; g < G; g++) {
      float lb = bounds[(size_t)N * (1 + g) + i] - maxdrift[g];
      bounds[(size_t)N * (1 + g) + i] = lb;
      if (lb < minlb) minlb = lb;
    }
    if (minlb >= ub) { bounds[i] = ub; continue; }
    ntight++;
    ub = ko_distance(metric, X + (size_t)i * D, C + (size_t)a * D, D);
    bounds[i] = ub;
    if (minlb >= ub) continue;
    passed[npassed++] = i;
  }
  uint32_t ch = 0;
#pragma omp parallel for schedule(dynamic, 64) reduction(+ : ch)
  for (uint32_t pi = 0; pi < npassed; pi++) {
    uint32_t i = passed[pi];
    float ub = bounds[i];
    uint32_t a = assign[i];
    float mn = ub, sec = FLT_MAX;
    uint32_t near = a;
    for (uint32_t c = 0; c < K; c++) {
      if (c == a) continue;
      uint32_t g = groups[c];
      if (g >= G) continue;
      float lb = bounds[(size_t)N * (1 + g) + i];
      if (lb >= ub) { if (lb < sec) sec = lb; continue; }
      lb += maxdrift[g] - drift[c];
      if (sec < lb) continue;
      float d = ko_distance(metric, X + (size_t)i * D, C + (size_t)c * D, D);
      if (d < mn) { sec = mn; mn = d; near = c; }
      else if (d < sec) sec = d;
    }
    uint32_t ng = groups[near], pg = groups[a];
    if (ng < G) bounds[(size_t)N * (1 + ng) + i] = sec; /* deviation: ng < G, pg < G (yy_finish_kernel) */
    if (ng != pg && pg < G) {
      float pb = bounds[(size_t)N * (1 + pg) + i];
      if (pb > ub) bounds[(size_t)N * (1 + pg) + i] = ub;
    }
    bounds[i] = mn;
    if (a != near) { assign[i] = near; ch++; }
  }
  free(passed);
  if (tight_out) *tight_out = ntight;
  if (passed_out) *passed_out = npassed;
  return ch;
}

/* ------------------------------------------------------------------------------------------ */
/* Whole k-means run from imported centroids: kmeans_cuda_yy, kmeans.cu:1028-1263.              */
/* yy_groups==0 or tolerance>=0.11 -> pure Lloyd.  Returns total "iteration" lines emitted.     */
/* ------------------------------------------------------------------------------------------ */
int ko_kmeans(int metric, float tolerance, uint32_t yy_groups, const float *X, uint32_t N, int D,
              uint32_t K, float *C, uint32_t *assign, int log, int max_iter) {
  uint32_t *prev = (uint32_t *)malloc(sizeof(uint32_t) * N);
  uint32_t *ccounts = (uint32_t *)malloc(sizeof(uint32_t) * K);
  int lines = 0;
  if (yy_groups == 0 || 0.11f <= tolerance) {
    lines = ko_lloyd_loop(metric, tolerance, X, N, D, K, C, ccounts, prev, assign, log, NULL, max_iter);
    free(prev); free(ccounts);
    return lines;
  }
  uint32_t changed = 0;
  int iter = ko_lloyd_loop(metric, 0.11f, X, N, D, K, C, ccounts, prev, assign, log, &changed, max_iter);
  lines = iter;
  if ((float)changed <= tolerance * (float)N || (max_iter > 0 && iter >= max_iter)) {
    free(prev); free(ccounts);
    return lines;
  }
  /* group the centroids: k-means++ (srand(0)) + Lloyd to 2 % on the K x D centroid table,
   * kmeans.cu:1061-1094 */
  uint32_t G = yy_groups;
  float *GC = (float *)malloc(sizeof(float) * (size_t)G * D);
  uint32_t *groups = (uint32_t *)malloc(sizeof(uint32_t) * K);
  {
    uint32_t *gprev = (uint32_t *)malloc(sizeof(uint32_t) * K);
    uint32_t *gcnt = (uint32_t *)malloc(sizeof(uint32_t) * G);
    srand(0);
    ko_init_plusplus(metric, C, K, D, G, GC);
    lines += ko_lloyd_loop(metric, 0.02f, C, K, D, G, GC, gcnt, gprev, groups, log, NULL, 0);
    free(gprev); free(gcnt);
  }
  float *bounds = (float *)malloc(sizeof(float) * (size_t)N * (G + 1));
  float *oldC = (float *)malloc(sizeof(float) * (size_t)K * D);
  float *drift = (float *)malloc(sizeof(float) * K);
  float *maxdrift = (float *)malloc(sizeof(float) * G);
  int refresh = 1;
  uint32_t npassed = 0;
  changed = 0; /* prepare_mem(resume=true) zeroes d_changed_number, kmeans.cu:1102-1103 */
  for (;; iter++) {
    if (!refresh) {
      if (log) printf("iteration %d: %u reassignments\n", iter, changed);
      lines++;
      if ((float)changed <= tolerance * (float)N) break;
      if (max_iter > 0 && lines >= max_iter) break;
      changed = 0;
      if (1.f - (npassed + 0.f) / N < 1e-4f) refresh = 1;
      npassed = 0;
    }
    if (refresh) {
      ko_yy_init(metric, X, C, N, D, K, G, groups, assign, bounds);
      refresh = 0;
    }
    memcpy(oldC, C, sizeof(float) * (size_t)K * D);
    ko_adjust(metric, X, N, D, K, prev, assign, C, ccounts);
    ko_yy_drifts(metric, C, oldC, K, D, G, groups, drift, maxdrift);
    changed = ko_yy_step(metric, X, C, N, D, K, G, groups, drift, maxdrift, assign, prev, bounds, NULL, &npassed);
  }
  free(prev); free(ccounts); free(GC); free(groups); free(bounds); free(oldC); free(drift);
  free(maxdrift);
  return lines;
}

/* distance accumulated chunk-wise the way knn.cu:36-47 / :79-100 do: a fresh Kahan sum per
 * feature chunk (partial / partial_t, metric_abstraction.h:103-136, 224-248), chunks added with a
 * plain fp32 '+=' into a zeroed accumulator, finalize (sqrt / clamped acos) at the end. */
float ko_chunked_distance(int metric, const float *a, const float *b, int D, int chunk) {
  float acc = 0.f;
  for (int f0 = 0; f0 < D; f0 += chunk) {
    int n = D - f0 < chunk ? D - f0 : chunk;
    float part = (metric == KO_COS) ? ko_kahan_dot(a + f0, b + f0, n) : ko_sqdiff(a + f0, b + f0, n);
    acc += part;
  }
  return (metric == KO_COS) ? ko_acos_clamped(acc) : sqrtf(acc);
}

/* ------------------------------------------------------------------------------------------ */
/* k-NN: knn.cu:19-131 (radii, centroid distance matrix), :133-243 (search), host prep          */
/* kmcuda.cc:648-691.  Output: k neighbour indices per sample ascending by distance, self       */
/* excluded.  Heap semantics restated as "keep the k smallest with '<=' replacement", emitted   */
/* by repeatedly popping the max (knn.cu:239-242).                                              */
/* ------------------------------------------------------------------------------------------ */
static void ko_push(int k, float dist, uint32_t index, float *hd, uint32_t *hi) { /* knn.cu:133-175 */
  int pos = 0;
  for (;;) {
    float left = 0, right = 0;
    int left_le, right_le;
    if (2 * pos + 1 < k) { left = hd[2 * pos + 1]; left_le = dist >= left; } else left_le = 1;
    if (2 * pos + 2 < k) { right = hd[2 * pos + 2]; right_le = dist >= right; } else right_le = 1;
    if (left_le && right_le) { hd[pos] = dist; hi[pos] = index; return; }
    int go_right;
    if (!left_le && !right_le) go_right = (left <= right);
    else go_right = left_le;
    int child = go_right ? 2 * pos + 2 : 2 * pos + 1;
    hd[pos] = hd[child]; hi[pos] = hi[child];
    pos = child;
  }
}

typedef struct { uint32_t a, i; } ko_pair;
static int ko_pair_cmp(const void *x, const void *y) {
  const ko_pair *p = (const ko_pair *)x, *q = (const ko_pair *)y;
  if (p->a != q->a) return p->a < q->a ? -1 : 1;
  return p->i < q->i ? -1 : (p->i > q->i);
}

/* query_idx==NULL -> all N samples are queries; else nq rows listed in query_idx.
 * out is [nq][k]; frac_out (optional) = evaluated pairs / N^2-ish counter of knn.cu:521-530. */
void ko_knn(int metric, int k, const float *X, uint32_t N, int D, const float *C, uint32_t K,
            const uint32_t *assign, const uint32_t *query_idx, uint32_t nq, uint32_t *out,
            double *pairs_out) {
  ko_pair *pairs = (ko_pair *)malloc(sizeof(ko_pair) * N);
  for (uint32_t s = 0; s < N; s++) { pairs[s].a = assign[s]; pairs[s].i = s; }
  qsort(pairs, N, sizeof(ko_pair), ko_pair_cmp);
  uint32_t *inv = (uint32_t *)malloc(sizeof(uint32_t) * N);
  uint32_t *off = (uint32_t *)calloc(K + 2, sizeof(uint32_t));
  for (uint32_t s = 0; s < N; s++) { inv[s] = pairs[s].i; if (pairs[s].a < K) off[pairs[s].a + 1]++; }
  for (uint32_t c = 0; c < K; c++) off[c + 1] += off[c];
  free(pairs);
  float *R = (float *)malloc(sizeof(float) * K);
  float *Cd = (float *)malloc(sizeof(float) * (size_t)K * K);
  for (uint32_t c = 0; c < K; c++) { /* knn.cu:19-58: partial sums over 16-feature chunks */
    float m = -1;
    for (uint32_t p = off[c]; p < off[c + 1]; p++) {
      float d = ko_chunked_distance(metric, X + (size_t)inv[p] * D, C + (size_t)c * D, D, 16);
      if (d > m) m = d;
    }
    R[c] = m > -1 ? m : NAN;
  }
#pragma omp parallel for schedule(static)
  for (uint32_t a = 0; a < K; a++) /* knn.cu:60-131: 24-feature chunks, then mirrored */
    for (uint32_t b = 0; b < K; b++)
      Cd[(size_t)a * K + b] = ko_chunked_distance(metric, C + (size_t)a * D, C + (size_t)b * D, D, 24);
  uint32_t Q = query_idx ? nq : N;
  double total_pairs = 0;
#pragma omp parallel for schedule(dynamic, 16) reduction(+ : total_pairs)
  for (uint32_t qi = 0; qi < Q; qi++) {
    uint32_t s = query_idx ? query_idx[qi] : qi;
    float *hd = (float *)malloc(sizeof(float) * k);
    uint32_t *hi = (uint32_t *)malloc(sizeof(uint32_t) * k);
    for (int i = 0; i < k; i++) { hd[i] = FLT_MAX; hi[i] = UINT32_MAX; }
    uint32_t A = assign[s];
    const float *xs = X + (size_t)s * D;
    float dA = ko_distance(metric, xs, C + (size_t)A * D, D);
    float kth = FLT_MAX;
    total_pairs += off[A + 1] - off[A];
    for (uint32_t p = off[A]; p < off[A + 1]; p++) {
      uint32_t o = inv[p];
      if (o == s) continue;
      float d = ko_distance(metric, xs, X + (size_t)o * D, D);
      if (d <= kth) { ko_push(k, d, o, hd, hi); kth = hd[0]; }
    }
    for (uint32_t B = 0; B < K; B++) {
      if (B == A) continue;
      float cd = Cd[(size_t)B * K + A];
      if (cd != cd) continue;
      if (cd - dA - R[B] > kth) continue;
      total_pairs += off[B + 1] - off[B];
      for (uint32_t p = off[B]; p < off[B + 1]; p++) {
        uint32_t o = inv[p];
        float d = ko_distance(metric, xs, X + (size_t)o * D, D);
        if (d <= kth) { ko_push(k, d, o, hd, hi); kth = hd[0]; }
      }
    }
    for (int i = k - 1; i >= 0; i--) {
      out[(size_t)qi * k + i] = hi[0];
      ko_push(k, -1.f, UINT32_MAX, hd, hi);
    }
    free(hd); free(hi);
  }
  if (pairs_out) *pairs_out = total_pairs;
  free(inv); free(off); free(R); free(Cd);
}

/* round-down FMA through the FP environment: used only by the self-test that validates ko_fma_rd */
#include <fenv.h>
float ko_fma_rd_fenv(float a, float b, float c) {
  volatile float va = a, vb = b, vc = c;
  int old = fegetround();
  fesetround(FE_DOWNWARD);
  volatile float r = fmaf(va, vb, vc);
  fesetround(old);
  return r;
}
