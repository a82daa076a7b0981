// seeding.cu -- a Job's centroid initialisation (reference kmcuda.cc:189-400): import, random, k-means++, AFK-MC2, k-means||,
// greedy k-means++.
#include <random>

#include "job.h"

namespace kmb {

// a seeding pick that landed on a zero-weight row moves to the next positive-weight row (the previous one at the end);
// the same rule as skip_zero_weight in simt_kernels.cu
static uint32_t skip_zero_weight_host(const std::vector<float>& w, uint32_t s) {
  if (w.empty() || w[s] > 0.f) return s;
  for (uint32_t u = s + 1; u < w.size(); u++)
    if (w[u] > 0.f) return u;
  for (uint32_t u = s; u-- > 0;)
    if (w[u] > 0.f) return u;
  return s;
}

KMCUDAResult Job::set_centroids_from_host(const float* hostC) {
  for (auto& d : devs) {
    KMB_CU(cudaSetDevice(d.dev), kmcudaRuntimeError);
    KMB_CU(cudaMemcpyAsync(d.C.get(), hostC, sizeof(float) * static_cast<size_t>(K) * D,
                           cudaMemcpyHostToDevice, d.st), kmcudaMemoryCopyError);
  }
  return sync_all();
}

KMCUDAResult Job::fetch_row(uint32_t idx, float* host_row) {
  for (auto& d : devs) {
    if (idx >= d.off && idx < d.off + d.len) {
      KMB_CU(cudaSetDevice(d.dev), kmcudaRuntimeError);
      KMB_CU(cudaMemcpy(host_row, d.X.get() + static_cast<size_t>(idx - d.off) * D, sizeof(float) * D,
                        cudaMemcpyDeviceToHost), kmcudaMemoryCopyError);
      return kmcudaSuccess;
    }
  }
  return kmcudaRuntimeError;
}

// identity permutation of N rows shuffled with rand() the way libstdc++'s std::random_shuffle does (kmcuda.cc:245-260)
static std::vector<uint32_t> random_order(uint32_t N) {
  std::vector<uint32_t> chosen(N);
  for (uint32_t s = 0; s < N; s++) chosen[s] = s;
  for (uint32_t i = 1; i < N; i++) {
    uint32_t j = static_cast<uint32_t>(rand() % (static_cast<int64_t>(i) + 1));
    if (i != j) std::swap(chosen[i], chosen[j]);
  }
  return chosen;
}

// The shuffled walk of init_random: hostC rows start .. K - 1 are the rows of random_order(N) (the rand() draws after
// the caller's srand) in walk order, skipping rows of weight 0 and those marked in `taken`.  `what` prefixes the
// message when the walk runs out of rows.
KMCUDAResult Job::fill_random(float* hostC, uint32_t start, const std::vector<char>* taken, const char* what) {
  KMB_RET(load_host_weights());
  const std::vector<uint32_t> order = random_order(N);
  uint32_t c = start;
  for (uint32_t s = 0; s < N && c < K; s++) {
    const uint32_t i = order[s];
    if ((taken && (*taken)[i]) || (weighted && !(host_w[i] > 0.f))) continue;
    KMB_RET(fetch_row(i, hostC + static_cast<size_t>(c) * D));
    c++;
  }
  if (c < K) {
    KMB_INFO("%s: only %" PRIu32 " samples have a positive weight, %" PRIu32 " clusters\n", what, c, K);
    return kmcudaInvalidArguments;
  }
  return kmcudaSuccess;
}

// K distinct random samples; same host RNG walk as the reference (kmcuda.cc:245-260).
// Weighted: the walk over the shuffled order skips rows of weight 0.
KMCUDAResult Job::init_random() {
  KMB_INFO("randomly picking initial centroids...\n");
  std::vector<float> hostC(static_cast<size_t>(K) * D);
  KMB_RET(fill_random(hostC.data(), 0, nullptr, "random init"));
  return set_centroids_from_host(hostC.data());
}

// first centroid of k-means++ / AFK-MC2: rand() % N, re-drawn while the row is NaN (kmcuda.cc:270-276) or has weight 0
KMCUDAResult Job::draw_first_centroid(float* hostC, uint32_t* first_out) {
  KMB_RET(load_host_weights());
  uint32_t first_index;
  float smoke = NAN;
  do {
    first_index = rand() % N;
    if (weighted && !(host_w[first_index] > 0.f)) continue;   // (smoke stays NaN: draw again)
    std::vector<float> row(D);
    KMB_RET(fetch_row(first_index, row.data()));
    smoke = row[0];
    if (smoke == smoke) memcpy(hostC, row.data(), sizeof(float) * D);
  } while (smoke != smoke);
  *first_out = first_index;
  return kmcudaSuccess;
}

// k-means++ driven by the host RNG: reference kmcuda.cc:262-333 + kernel kmeans.cu:42-67.  Weighted: the draw is
// proportional to w * d (the reference's d, not d^2, times the weight)
KMCUDAResult Job::init_plusplus() {
  std::vector<float> hostC(static_cast<size_t>(K) * D);
  std::vector<float> host_dists(N);
  uint32_t first_index;
  KMB_RET(draw_first_centroid(hostC.data(), &first_index));
  KMB_INFO("performing kmeans++...\n");
  {
    const char* hp = getenv("KMCUDA_B200_HOST_PLUSPLUS");   // A/B: the reference-shaped host loop below
    if (devs.size() == 1 && !(hp && hp[0] == '1')) {
      // device-resident rounds: no D2H of the distances, no host walk, no H2D of the chosen row; the draws are the
      // reference's rand() sequence (one per round, kmcuda.cc:296)
      Dev& d = devs[0];
      KMB_CU(cudaSetDevice(d.dev), kmcudaRuntimeError);
      const uint32_t nb = (d.len + 255) / 256;
      DevBuf<double> bsum, bpre;
      DevBuf<uint32_t> chosen;
      Drain drain{*this};
      KMB_CU(d.dists.alloc(d.len), kmcudaMemoryAllocationFailure);
      KMB_CU(bsum.alloc(static_cast<size_t>(nb) + 1), kmcudaMemoryAllocationFailure);
      KMB_CU(bpre.alloc(static_cast<size_t>(nb) + 1), kmcudaMemoryAllocationFailure);
      KMB_CU(chosen.alloc(K), kmcudaMemoryAllocationFailure);
      KMB_CU(cudaMemcpyAsync(d.C.get(), hostC.data(), sizeof(float) * D, cudaMemcpyHostToDevice, d.st), kmcudaMemoryCopyError);
      for (uint32_t i = 1; i < K; i++) {
        const double choice = ((rand() + .0) / RAND_MAX);
        KMB_CU(launch_plusplus_round(metric, d.X, d.len, D, d.C.get(), i, choice, d.dists, bsum, bpre, chosen, d.st,
                                     d.w.get()), kmcudaRuntimeError);
        if ((i & 255) == 0) KMB_CU(cudaStreamSynchronize(d.st), kmcudaRuntimeError);   // keep the launch queue shallow
      }
      KMB_CU(cudaStreamSynchronize(d.st), kmcudaRuntimeError);
      d.dists.release();
      return kmcudaSuccess;
    }
  }
  for (auto& d : devs) {
    KMB_CU(cudaSetDevice(d.dev), kmcudaRuntimeError);
    KMB_CU(d.dists.alloc(d.len), kmcudaMemoryAllocationFailure);
  }
  for (uint32_t i = 1; i < K; i++) {
    if (verbosity > 1 || (verbosity > 0 && (K < 100 || i % (K / 100) == 0))) {
      printf("\rstep %d", i);
      fflush(stdout);
    }
    for (auto& d : devs) {
      KMB_CU(cudaSetDevice(d.dev), kmcudaRuntimeError);
      float* cdst = d.C.get() + static_cast<size_t>(i - 1) * D;
      KMB_CU(cudaMemcpyAsync(cdst, hostC.data() + static_cast<size_t>(i - 1) * D, sizeof(float) * D,
                             cudaMemcpyHostToDevice, d.st), kmcudaMemoryCopyError);
      KMB_CU(cudaMemsetAsync(d.d_dsum.get(), 0, sizeof(double), d.st), kmcudaRuntimeError);
      KMB_CU(launch_plusplus_step(metric, d.X, d.len, D, cdst, i == 1, d.dists, d.d_dsum, d.st, d.w.get()),
             kmcudaRuntimeError);
      KMB_CU(cudaMemcpyAsync(host_dists.data() + d.off, d.dists.get(), sizeof(float) * d.len,
                             cudaMemcpyDeviceToHost, d.st), kmcudaMemoryCopyError);
    }
    std::vector<double> parts;
    KMB_RET(gather([&](size_t s) { return devs[s].d_dsum.get(); }, &parts));
    double dist_sum = 0;
    for (double part : parts) dist_sum += part;
    if (weighted)   // the walk below runs over w * d, the mass the device summed (dists[] on the device keep d)
      for (uint32_t s = 0; s < N; s++) host_dists[s] *= host_w[s];
    if (dist_sum != dist_sum) KMB_INFO("\ninternal bug inside kmeans_init_centroids: dist_sum is NaN\n");
    double choice = ((rand() + .0) / RAND_MAX);
    uint32_t choice_approx = static_cast<uint32_t>(choice * N);
    double choice_sum = choice * dist_sum;
    uint32_t j;
    if (choice_approx < 100) {
      double s2 = 0;
      for (j = 0; j < N && s2 < choice_sum; j++) s2 += host_dists[j];
    } else {
      double s2 = 0;
      for (uint32_t t = 0; t < choice_approx; t++) s2 += host_dists[t];
      if (s2 < choice_sum) {
        for (j = choice_approx; j < N && s2 < choice_sum; j++) s2 += host_dists[j];
      } else {
        for (j = choice_approx; j > 1 && s2 >= choice_sum; j--) s2 -= host_dists[j];
        j++;
      }
    }
    if (j == 0 || j > N) {
      KMB_INFO("\ninternal bug in kmeans_init_centroids: j = %" PRIu32 "\n", j);
      j = std::min(std::max(j, 1u), N);
    }
    if (weighted) j = 1 + skip_zero_weight_host(host_w, j - 1);
    KMB_RET(fetch_row(j - 1, hostC.data() + static_cast<size_t>(i) * D));
  }
  for (auto& d : devs) d.dists.release();
  return set_centroids_from_host(hostC.data());
}

// AFK-MC2 (Bachem et al. 2016; reference kmcuda.cc:337-396, kernels kmeans.cu:69-212): proposal distribution
// q = 1/(2N) + d(x, c0)^2 / (2 sum d^2), then for every further centroid a Markov chain of length m over
// candidates drawn from q, accepting with probability min(1, (p'/q')/(p/q)) where p = squared distance to the
// nearest chosen centroid.  The reference draws candidates and acceptance thresholds with cuRAND on the device;
// here the chain is driven by a host generator seeded with `seed` (deterministic per seed; the reference's own q
// depends on float atomics, so its runs are only statistically reproducible as well).  The distance work (q and
// the candidates' nearest-centroid distances) runs on the shards that own the samples.
//
// Weighted: q = w / (2 W) + w d^2 / (2 sum w d^2) and p = w * (squared distance), so zero-weight rows are never drawn.
// Rows whose distance to c0 is not finite (a NaN feature, the first one included) have q = 0 and add nothing to
// sum w d^2: they are never drawn either.  Drawn, such a row would have no finite distance to any centroid, p = +inf,
// and the chain would always take it.
KMCUDAResult Job::init_afkmc2(uint32_t m, uint32_t seed) {
  std::vector<float> hostC(static_cast<size_t>(K) * D);
  std::vector<float> host_dists(N);
  uint32_t first_index;
  KMB_RET(draw_first_centroid(hostC.data(), &first_index));   // kmcuda.cc:346-353
  KMB_INFO("afkmc2: calculating q (c0 = %" PRIu32 ")... ", first_index);
  for (auto& d : devs) {
    KMB_CU(cudaSetDevice(d.dev), kmcudaRuntimeError);
    KMB_CU(d.dists.alloc(std::max<size_t>(d.len, 2 * static_cast<size_t>(m))), kmcudaMemoryAllocationFailure);
    KMB_CU(cudaMemcpyAsync(d.C.get(), hostC.data(), sizeof(float) * D, cudaMemcpyHostToDevice, d.st), kmcudaMemoryCopyError);
    KMB_CU(cudaMemsetAsync(d.d_dsum.get(), 0, sizeof(double), d.st), kmcudaRuntimeError);
    KMB_CU(launch_plusplus_step(metric, d.X, d.len, D, d.C.get(), 1, d.dists, d.d_dsum, d.st, nullptr, NAN),
           kmcudaRuntimeError);
    KMB_CU(cudaMemcpyAsync(host_dists.data() + d.off, d.dists.get(), sizeof(float) * d.len, cudaMemcpyDeviceToHost, d.st),
           kmcudaMemoryCopyError);
  }
  KMB_RET(sync_all());
  std::vector<float> q(N);
  std::vector<double> cdf(N);
  {
    // (unweighted: w = 1 and W = N)
    const double W = weighted ? wtotal : static_cast<double>(N);
    double dsum = 0;
    for (uint32_t i = 0; i < N; i++) {
      const double d2 = static_cast<double>(host_dists[i]) * host_dists[i];
      if (std::isfinite(d2)) dsum += weighted ? host_w[i] * d2 : d2;
    }
    double acc = 0;
    for (uint32_t i = 0; i < N; i++) {
      const double d2 = static_cast<double>(host_dists[i]) * host_dists[i];
      const double wi = weighted ? host_w[i] : 1.0;
      const double qi = !std::isfinite(d2) ? 0.0
                        : wi / (2.0 * W) + (dsum > 0 ? wi * d2 / (2.0 * dsum) : wi / (2.0 * W));
      q[i] = static_cast<float>(qi);
      acc += qi;
      cdf[i] = acc;
    }
  }
  KMB_INFO("done\n");
  std::mt19937_64 gen(seed);
  auto uniform = [&gen]() { return (static_cast<double>(gen() >> 11) + 0.5) * (1.0 / 9007199254740992.0); };
  std::vector<uint32_t> cand(m), local(m);
  std::vector<float> p_cand(m), rand_a(m);
  struct Scratch { DevBuf<uint32_t> rows; DevBuf<float> mind; std::vector<uint32_t> slots; std::vector<float> host; };
  std::vector<Scratch> sc(devs.size());
  Drain drain{*this};
  for (size_t i = 0; i < devs.size(); i++) {
    KMB_CU(cudaSetDevice(devs[i].dev), kmcudaRuntimeError);
    KMB_CU(sc[i].rows.alloc(m), kmcudaMemoryAllocationFailure);
    KMB_CU(sc[i].mind.alloc(m), kmcudaMemoryAllocationFailure);
    sc[i].host.resize(m);
  }
  for (uint32_t k = 1; k < K; k++) {
    if (verbosity > 1 || (verbosity > 0 && (K < 100 || k % (K / 100) == 0))) {
      printf("\rstep %d", k);
      fflush(stdout);
    }
    for (uint32_t j = 0; j < m; j++) {   // kmeans_afkmc2_random_step: first index whose cumulative q reaches the draw
      const double part = uniform() * cdf[N - 1];
      cand[j] = static_cast<uint32_t>(std::min<size_t>(std::lower_bound(cdf.begin(), cdf.end(), part) - cdf.begin(), N - 1));
      rand_a[j] = static_cast<float>(uniform());
    }
    for (size_t i = 0; i < devs.size(); i++) {
      Dev& d = devs[i];
      sc[i].slots.clear();
      uint32_t cnt = 0;
      for (uint32_t j = 0; j < m; j++)
        if (cand[j] >= d.off && cand[j] < d.off + d.len) {
          local[cnt++] = cand[j] - d.off;
          sc[i].slots.push_back(j);
        }
      if (cnt == 0) continue;
      KMB_CU(cudaSetDevice(d.dev), kmcudaRuntimeError);
      KMB_CU(cudaMemcpyAsync(sc[i].rows.get(), local.data(), sizeof(uint32_t) * cnt, cudaMemcpyHostToDevice, d.st),
             kmcudaMemoryCopyError);
      KMB_CU(cudaStreamSynchronize(d.st), kmcudaRuntimeError);   // `local` is reused for the next shard
      KMB_CU(launch_afkmc2_min_dist(metric, d.X, d.C, D, k, sc[i].rows, cnt, sc[i].mind, d.st), kmcudaRuntimeError);
      KMB_CU(cudaMemcpyAsync(sc[i].host.data(), sc[i].mind.get(), sizeof(float) * cnt, cudaMemcpyDeviceToHost, d.st),
             kmcudaMemoryCopyError);
    }
    for (size_t i = 0; i < devs.size(); i++) {
      if (sc[i].slots.empty()) continue;
      KMB_CU(cudaSetDevice(devs[i].dev), kmcudaRuntimeError);
      KMB_CU(cudaStreamSynchronize(devs[i].st), kmcudaRuntimeError);
      for (size_t t = 0; t < sc[i].slots.size(); t++) {
        const float dmin = sc[i].host[t];
        const uint32_t slot = sc[i].slots[t];
        p_cand[slot] = weighted ? host_w[cand[slot]] * (dmin * dmin) : dmin * dmin;
      }
    }
    float curr_prob = 0;
    uint32_t curr_ind = 0;
    for (uint32_t j = 0; j < m; j++) {   // kmcuda.cc:382-389
      const float cand_prob = p_cand[j] / q[cand[j]];
      if (curr_prob == 0 || cand_prob / curr_prob > rand_a[j]) {
        curr_ind = j;
        curr_prob = cand_prob;
      }
    }
    float* dst = hostC.data() + static_cast<size_t>(k) * D;
    KMB_RET(fetch_row(cand[curr_ind], dst));
    for (auto& d : devs) {
      KMB_CU(cudaSetDevice(d.dev), kmcudaRuntimeError);
      KMB_CU(cudaMemcpyAsync(d.C.get() + static_cast<size_t>(k) * D, dst, sizeof(float) * D, cudaMemcpyHostToDevice, d.st),
             kmcudaMemoryCopyError);
    }
  }
  KMB_RET(sync_all());
  for (auto& d : devs) d.dists.release();
  return set_centroids_from_host(hostC.data());
}

// k-means|| (Bahmani et al., "Scalable K-Means++", VLDB 2012; DESIGN.md §4g).  c0 is k-means++'s first centroid; each
// of `rounds` rounds draws every row independently with probability l w_i d_i^2 / phi (l = 2K, d_i the true distance
// to the nearest candidate so far, phi = sum w_i d_i^2), runs one assignment pass against the round's new candidates
// only and lowers d_i where the winner is closer.  The candidates, weighted by the sample weight they are nearest to,
// are then clustered down to K by the library's own weighted k-means++ / Lloyd run; with at most K candidates they are
// the centroids and init_random's walk fills the rest.  Every shard draws its own rows with a counter hash of the
// global row index, so the draws do not depend on the device split.
KMCUDAResult Job::init_kmeans_parallel(uint32_t rounds, uint32_t seed) {
  std::vector<float> cand(D);          // the candidate rows in list order (round, row index), host copy
  std::vector<uint32_t> cand_rows(1);  // their global row indices
  KMB_RET(draw_first_centroid(cand.data(), &cand_rows[0]));
  struct Work {
    DevBuf<float> table, gathered;     // this round's candidates (all shards'), this shard's drawn rows
    DevBuf<uint32_t> nearest, idx, count;
    DevBuf<double> bsum, phi;
    DevBuf<uint8_t> flags;
    DevBuf<char> tmp;
    size_t tmp_bytes = 0;
    uint32_t nb = 0, drawn = 0;
  };
  std::vector<Work> wk(devs.size());
  Drain drain{*this};
  for (size_t s = 0; s < devs.size(); s++) {
    Dev& d = devs[s];
    Work& w = wk[s];
    KMB_CU(cudaSetDevice(d.dev), kmcudaRuntimeError);
    w.nb = kmp_blocks(d.len);
    w.tmp_bytes = kmp_select_bytes(d.len);
    KMB_CU(d.dists.alloc(d.len), kmcudaMemoryAllocationFailure);
    KMB_CU(w.nearest.alloc(d.len), kmcudaMemoryAllocationFailure);
    KMB_CU(w.idx.alloc(d.len), kmcudaMemoryAllocationFailure);
    KMB_CU(w.count.alloc(1), kmcudaMemoryAllocationFailure);
    KMB_CU(w.bsum.alloc(w.nb), kmcudaMemoryAllocationFailure);
    KMB_CU(w.phi.alloc(1), kmcudaMemoryAllocationFailure);
    KMB_CU(w.flags.alloc(d.len), kmcudaMemoryAllocationFailure);
    KMB_CU(w.tmp.alloc(w.tmp_bytes), kmcudaMemoryAllocationFailure);
    KMB_CU(w.table.alloc(D), kmcudaMemoryAllocationFailure);
    KMB_CU(cudaMemcpyAsync(w.table.get(), cand.data(), sizeof(float) * D, cudaMemcpyHostToDevice, d.st),
           kmcudaMemoryCopyError);
    KMB_CU(launch_kmp_update(metric, d.X, d.len, D, w.table, 1, nullptr, 0, d.dists, w.nearest, d.w.get(), w.bsum, d.st),
           kmcudaRuntimeError);
    KMB_CU(launch_fixed_sum(w.bsum, w.nb, w.phi, d.st), kmcudaRuntimeError);
  }
  const double ell = 2.0 * K;
  for (uint32_t r = 1; r <= rounds; r++) {
    std::vector<double> parts;
    KMB_RET(gather([&](size_t s) { return wk[s].phi.get(); }, &parts));
    double phi = 0;
    for (double part : parts) phi += part;   // device order: the same total on every run
    if (!(phi > 0)) break;   // every row sits on a candidate
    for (size_t s = 0; s < devs.size(); s++) {
      Dev& d = devs[s];
      Work& w = wk[s];
      KMB_CU(cudaSetDevice(d.dev), kmcudaRuntimeError);
      KMB_CU(launch_kmp_draw(d.dists, d.w.get(), d.len, d.off, seed, r, ell, phi, w.flags, w.idx, w.count, w.tmp,
                             w.tmp_bytes, d.st), kmcudaRuntimeError);
    }
    std::vector<uint32_t> drawn;
    KMB_RET(gather([&](size_t s) { return wk[s].count.get(); }, &drawn));
    const uint32_t base = static_cast<uint32_t>(cand_rows.size());
    uint32_t fresh = 0;
    for (size_t s = 0; s < devs.size(); s++) {
      wk[s].drawn = drawn[s];
      fresh += drawn[s];
    }
    KMB_INFO("k-means|| round %" PRIu32 ": %" PRIu32 " candidates, cost %.17g\n", r, fresh, phi);
    if (fresh == 0) continue;   // nothing changes: the next round draws again from the same d
    // gather each shard's drawn rows, then every device gets the whole round's table in device (= row) order
    cand_rows.resize(base + fresh);
    for (size_t s = 0, at = base; s < devs.size(); s++) {
      Dev& d = devs[s];
      Work& w = wk[s];
      if (w.drawn == 0) continue;
      KMB_CU(cudaSetDevice(d.dev), kmcudaRuntimeError);
      KMB_CU(w.gathered.alloc(static_cast<size_t>(w.drawn) * D), kmcudaMemoryAllocationFailure);
      KMB_CU(launch_kmp_gather(d.X, D, w.idx, w.drawn, w.gathered, d.st), kmcudaRuntimeError);
      KMB_CU(cudaMemcpyAsync(cand_rows.data() + at, w.idx.get(), sizeof(uint32_t) * w.drawn, cudaMemcpyDeviceToHost,
                             d.st), kmcudaMemoryCopyError);
      at += w.drawn;
    }
    KMB_RET(sync_all());
    for (size_t s = 0, at = base; s < devs.size(); s++) {
      for (uint32_t j = 0; j < wk[s].drawn; j++) cand_rows[at + j] += devs[s].off;
      at += wk[s].drawn;
    }
    for (size_t t = 0; t < devs.size(); t++) {
      Dev& d = devs[t];
      KMB_CU(cudaSetDevice(d.dev), kmcudaRuntimeError);
      KMB_CU(wk[t].table.alloc(static_cast<size_t>(fresh) * D), kmcudaMemoryAllocationFailure);
      size_t at = 0;
      for (size_t s = 0; s < devs.size(); s++) {
        if (wk[s].drawn == 0) continue;
        KMB_CU(cudaMemcpyPeerAsync(wk[t].table.get() + at * D, d.dev, wk[s].gathered.get(), devs[s].dev,
                                   sizeof(float) * wk[s].drawn * D, d.st), kmcudaMemoryCopyError);
        at += wk[s].drawn;
      }
    }
    cand.resize(static_cast<size_t>(base + fresh) * D);
    KMB_CU(cudaSetDevice(devs[0].dev), kmcudaRuntimeError);
    KMB_CU(cudaMemcpyAsync(cand.data() + static_cast<size_t>(base) * D, wk[0].table.get(),
                           sizeof(float) * static_cast<size_t>(fresh) * D, cudaMemcpyDeviceToHost, devs[0].st),
           kmcudaMemoryCopyError);
    KMB_RET(sync_all());   // (the peer copies have read every `gathered` buffer)
    // one assignment pass of every shard against the round's candidates, then the running-minimum update
    std::vector<std::unique_ptr<Shard>> pass(devs.size());
    for (size_t s = 0; s < devs.size(); s++) {
      Dev& d = devs[s];
      Work& w = wk[s];
      pass[s].reset(new Shard(metric, d.dev, d.len, D, fresh, verbosity));
      KMB_RET(pass[s]->create(false));
      KMB_CU(cudaSetDevice(d.dev), kmcudaRuntimeError);
      KMB_CU(cudaMemsetAsync(d.assign.get(), 0xff, sizeof(uint32_t) * d.len, d.st), kmcudaRuntimeError);
      KMB_RET(pass[s]->assign(d.len, d.X, w.table, d.assign, d.prev, d.d_changed, d.st));
      KMB_CU(launch_kmp_update(metric, d.X, d.len, D, w.table, fresh, d.assign, base, d.dists, w.nearest, d.w.get(),
                               w.bsum, d.st), kmcudaRuntimeError);
      KMB_CU(launch_fixed_sum(w.bsum, w.nb, w.phi, d.st), kmcudaRuntimeError);
    }
    KMB_RET(sync_all());
    for (auto& p : pass) KMB_RET(p->check_pipeline());
  }
  const uint32_t Cn = static_cast<uint32_t>(cand_rows.size());
  KMB_INFO("k-means||: %" PRIu32 " candidates -> %" PRIu32 " centroids\n", Cn, K);
  g_prof.mark("init: k-means|| rounds");
  std::vector<float> hostC(static_cast<size_t>(K) * D);
  if (Cn <= K) {
    // the candidates, then init_random's walk from srand(seed) over the rows not chosen yet (and of positive weight)
    memcpy(hostC.data(), cand.data(), sizeof(float) * static_cast<size_t>(Cn) * D);
    std::vector<char> taken(N, 0);
    for (uint32_t i : cand_rows) taken[i] = 1;
    srand(seed);
    KMB_RET(fill_random(hostC.data(), Cn, &taken, "k-means||"));
    for (auto& d : devs) d.dists.release();
    KMB_RET(set_centroids_from_host(hostC.data()));
    g_prof.mark("init: k-means|| recluster");
    return kmcudaSuccess;
  }
  // candidate weights W_j = sum of w_i over the rows nearest to candidate j: exact counts, or compensated fp32 sums per
  // device added in device order (the weighted update's rule)
  std::vector<float> W(Cn, 0.f);
  {
    std::vector<uint32_t> total(Cn, 0), part_u(Cn);
    std::vector<float> part_f(Cn);
    for (size_t s = 0; s < devs.size(); s++) {
      Dev& d = devs[s];
      Work& w = wk[s];
      KMB_CU(cudaSetDevice(d.dev), kmcudaRuntimeError);
      if (weighted) {
        DevBuf<uint32_t> keys, start;
        DevBuf<float> wsorted, Wd;
        const size_t bytes = kmp_weights_bytes(d.len);
        KMB_CU(keys.alloc(d.len), kmcudaMemoryAllocationFailure);
        KMB_CU(start.alloc(2 * static_cast<size_t>(Cn)), kmcudaMemoryAllocationFailure);
        KMB_CU(wsorted.alloc(d.len), kmcudaMemoryAllocationFailure);
        KMB_CU(Wd.alloc(Cn), kmcudaMemoryAllocationFailure);
        KMB_CU(w.tmp.alloc(bytes), kmcudaMemoryAllocationFailure);
        KMB_CU(launch_kmp_weights(w.nearest, d.w, d.len, Cn, keys, wsorted, start, w.tmp, bytes, Wd, d.st),
               kmcudaRuntimeError);
        KMB_CU(cudaMemcpyAsync(part_f.data(), Wd.get(), sizeof(float) * Cn, cudaMemcpyDeviceToHost, d.st),
               kmcudaMemoryCopyError);
        KMB_CU(cudaStreamSynchronize(d.st), kmcudaRuntimeError);
        for (uint32_t j = 0; j < Cn; j++) W[j] += part_f[j];
      } else {
        DevBuf<uint32_t> counts;
        KMB_CU(counts.alloc(Cn), kmcudaMemoryAllocationFailure);
        KMB_CU(cudaMemsetAsync(counts.get(), 0, sizeof(uint32_t) * Cn, d.st), kmcudaRuntimeError);
        KMB_CU(launch_kmp_counts(w.nearest, d.len, counts, d.st), kmcudaRuntimeError);
        KMB_CU(cudaMemcpyAsync(part_u.data(), counts.get(), sizeof(uint32_t) * Cn, cudaMemcpyDeviceToHost, d.st),
               kmcudaMemoryCopyError);
        KMB_CU(cudaStreamSynchronize(d.st), kmcudaRuntimeError);
        for (uint32_t j = 0; j < Cn; j++) total[j] += part_u[j];
      }
    }
    if (!weighted)
      for (uint32_t j = 0; j < Cn; j++) W[j] = static_cast<float>(total[j]);
  }
  for (auto& d : devs) d.dists.release();
  wk.clear();
  // recluster: the steps of kmcuda_b200_kmeans_weighted(k-means++, tolerance 0.01, yinyang_t 0, metric, seed,
  // verbosity 0) on the candidate rows on the first device, with the same result.  Its phases stay out of the caller's
  // profile and log.  Two checks of the public call do not apply to the nested run:
  // - the unit-length probe of angular samples: the call's own samples passed it or were fp16x2, whose widened rows
  //   are unit length only to fp16 precision;
  // - KMCUDA_B200_STRICT_UPDATE=1, which replays the reference's unweighted update and would drop the weights W.
  {
    const bool prof = g_prof.on;
    g_prof.on = false;
    Job sub(metric, Cn, D, K, 0);
    sub.weighted = true;
    KMCUDAResult res = sub.setup({devs[0].dev});
    if (res == kmcudaSuccess) {
      sub.devs[0].shard->strict_update = false;
      res = sub.ingest(cand.data(), W.data(), -1, false);
    }
    if (res == kmcudaSuccess) res = sub.check_weights();
    if (res == kmcudaSuccess) {
      srand(seed);
      res = sub.init_plusplus();
    }
    if (res == kmcudaSuccess) res = sub.yinyang(0.01f, 0);
    g_prof.on = prof;
    KMB_RET(res);
    KMB_CU(cudaSetDevice(devs[0].dev), kmcudaRuntimeError);
    KMB_CU(cudaMemcpy(hostC.data(), sub.devs[0].C.get(), sizeof(float) * hostC.size(), cudaMemcpyDeviceToHost),
           kmcudaMemoryCopyError);
  }
  KMB_RET(set_centroids_from_host(hostC.data()));
  g_prof.mark("init: k-means|| recluster");
  return kmcudaSuccess;
}

// Greedy k-means++ (scikit-learn's _kmeans_plusplus; DESIGN.md §4m).  c0 is k-means++'s first centroid and d_i the true
// distance to it.  Each round r = 1 .. K - 1 draws L trial rows proportionally to m_i = w_i d_i^2 (trial t is the row
// with the smallest -ln u(seed, r, t, i) / m_i, an exponential race), computes for every trial the potential
// phi_t = sum mass(min(d_i, e_ti)) over the rows, e the true distance to the trial row, and keeps the trial of the
// smallest phi_t (the lowest t on equal values): its row becomes centroid r and d = min(d, e).  Chosen rows get d = 0.
// When no row has mass left, init_random's walk from srand(seed) fills the remaining centroids with rows not chosen yet.
// One GPU: every round stays on the device (greedy_plusplus.cu).  Several GPUs: each shard reduces its keys and its
// potential partials, and the host merges them in device order once per round.
KMCUDAResult Job::init_greedy_plusplus(uint32_t L, uint32_t seed) {
  std::vector<float> hostC(static_cast<size_t>(K) * D);
  std::vector<uint32_t> rows(K, UINT32_MAX);
  std::vector<double> pots(K, 0.0);
  KMB_RET(draw_first_centroid(hostC.data(), &rows[0]));
  KMB_INFO("greedy k-means++: %" PRIu32 " trials per round\n", L);
  struct Work {
    DevBuf<float> dprime, T;
    DevBuf<double> bkey, bsum, keys, phis, phi_log;
    DevBuf<uint32_t> brow, rows, row_log;
    DevBuf<GppCtl> ctl;
    std::vector<double> hkeys, hphis;
    std::vector<uint32_t> hrows;
  };
  std::vector<Work> wk(devs.size());
  Drain drain{*this};
  const bool single = devs.size() == 1;
  const GppCtl ctl0{UINT32_MAX, rows[0], 0, 0};   // round 1's draw sets d[c0] = 0
  for (size_t s = 0; s < devs.size(); s++) {
    Dev& d = devs[s];
    Work& w = wk[s];
    KMB_CU(cudaSetDevice(d.dev), kmcudaRuntimeError);
    KMB_CU(d.dists.alloc(std::max(d.len, 1u)), kmcudaMemoryAllocationFailure);
    KMB_CU(w.dprime.alloc(static_cast<size_t>(L) * std::max(d.len, 1u)), kmcudaMemoryAllocationFailure);
    KMB_CU(w.T.alloc(static_cast<size_t>(L) * D), kmcudaMemoryAllocationFailure);
    KMB_CU(w.bkey.alloc(static_cast<size_t>(L) * gpp_draw_blocks(d.len)), kmcudaMemoryAllocationFailure);
    KMB_CU(w.brow.alloc(static_cast<size_t>(L) * gpp_draw_blocks(d.len)), kmcudaMemoryAllocationFailure);
    KMB_CU(w.bsum.alloc(static_cast<size_t>(L) * gpp_trial_blocks(d.len)), kmcudaMemoryAllocationFailure);
    KMB_CU(w.keys.alloc(L), kmcudaMemoryAllocationFailure);
    KMB_CU(w.rows.alloc(L), kmcudaMemoryAllocationFailure);
    KMB_CU(w.phis.alloc(L), kmcudaMemoryAllocationFailure);
    KMB_CU(w.ctl.alloc(1), kmcudaMemoryAllocationFailure);
    w.hkeys.resize(L);
    w.hphis.resize(L);
    w.hrows.resize(L);
    if (single) {
      KMB_CU(w.row_log.alloc(K), kmcudaMemoryAllocationFailure);
      KMB_CU(w.phi_log.alloc(K), kmcudaMemoryAllocationFailure);
      KMB_CU(cudaMemsetAsync(w.row_log.get(), 0xff, sizeof(uint32_t) * K, d.st), kmcudaRuntimeError);
      KMB_CU(cudaMemcpyAsync(d.C.get(), hostC.data(), sizeof(float) * D, cudaMemcpyHostToDevice, d.st),
             kmcudaMemoryCopyError);
    }
    // d = the true distance to c0 (w.T's first row), kmp_update_kernel's start; its mass partials are not used
    KMB_CU(cudaMemcpyAsync(w.T.get(), hostC.data(), sizeof(float) * D, cudaMemcpyHostToDevice, d.st),
           kmcudaMemoryCopyError);
    KMB_CU(cudaMemcpyAsync(w.ctl.get(), &ctl0, sizeof(GppCtl), cudaMemcpyHostToDevice, d.st), kmcudaMemoryCopyError);
    KMB_CU(launch_kmp_update(metric, d.X, d.len, D, w.T, 1, nullptr, 0, d.dists, d.assign, d.w.get(), w.bsum, d.st),
           kmcudaRuntimeError);
  }
  uint32_t filled = K;   // the first centroid the fill walk provides (K: none)
  if (single) {
    Dev& d = devs[0];
    Work& w = wk[0];
    for (uint32_t r = 1; r < K; r++) {
      KMB_CU(launch_gpp_draw(d.dists, w.dprime, d.w.get(), d.len, d.off, L, w.ctl, gpp_round_key(seed, r), w.bkey,
                             w.brow, w.keys, w.rows, w.ctl, true, d.st), kmcudaRuntimeError);
      KMB_CU(launch_gpp_gather(d.X, d.off, D, w.rows, L, w.ctl, w.T, d.st), kmcudaRuntimeError);
      KMB_CU(launch_gpp_trial(metric, d.X, d.len, d.off, D, w.T, L, w.rows, d.dists, d.w.get(), w.ctl, w.dprime,
                              w.bsum, d.st), kmcudaRuntimeError);
      KMB_CU(launch_gpp_pick(w.bsum, d.len, L, w.ctl, w.rows, w.phis, true, d.X, d.off, D,
                             d.C.get() + static_cast<size_t>(r) * D, w.row_log.get() + r, w.phi_log.get() + r, d.st),
             kmcudaRuntimeError);
      if ((r & 255) == 0) KMB_CU(cudaStreamSynchronize(d.st), kmcudaRuntimeError);   // keep the launch queue shallow
    }
    std::vector<uint32_t> logged(K);
    KMB_CU(cudaMemcpyAsync(logged.data(), w.row_log.get(), sizeof(uint32_t) * K, cudaMemcpyDeviceToHost, d.st),
           kmcudaMemoryCopyError);
    KMB_CU(cudaMemcpyAsync(pots.data(), w.phi_log.get(), sizeof(double) * K, cudaMemcpyDeviceToHost, d.st),
           kmcudaMemoryCopyError);
    KMB_CU(cudaStreamSynchronize(d.st), kmcudaRuntimeError);
    for (uint32_t r = 1; r < K && filled == K; r++) {
      if (logged[r] == UINT32_MAX) filled = r;
      else rows[r] = logged[r];
    }
    if (filled < K)
      KMB_CU(cudaMemcpy(hostC.data(), d.C.get(), sizeof(float) * static_cast<size_t>(filled) * D,
                        cudaMemcpyDeviceToHost), kmcudaMemoryCopyError);
  } else {
    std::vector<float> trial(static_cast<size_t>(L) * D);
    std::vector<uint32_t> trows(L);
    for (uint32_t r = 1; r < K && filled == K; r++) {
      const uint64_t rkey = gpp_round_key(seed, r);
      for (size_t s = 0; s < devs.size(); s++) {
        Dev& d = devs[s];
        Work& w = wk[s];
        KMB_CU(cudaSetDevice(d.dev), kmcudaRuntimeError);
        KMB_CU(launch_gpp_draw(d.dists, w.dprime, d.w.get(), d.len, d.off, L, w.ctl, rkey, w.bkey, w.brow, w.keys,
                               w.rows, w.ctl, false, d.st), kmcudaRuntimeError);
        KMB_CU(cudaMemcpyAsync(w.hkeys.data(), w.keys.get(), sizeof(double) * L, cudaMemcpyDeviceToHost, d.st),
               kmcudaMemoryCopyError);
        KMB_CU(cudaMemcpyAsync(w.hrows.data(), w.rows.get(), sizeof(uint32_t) * L, cudaMemcpyDeviceToHost, d.st),
               kmcudaMemoryCopyError);
      }
      KMB_RET(sync_all());
      for (uint32_t t = 0; t < L; t++) {   // the minimum key, the lowest row on equal keys
        double k = INFINITY;
        uint32_t row = UINT32_MAX;
        for (const Work& w : wk)
          if (w.hkeys[t] < k || (w.hkeys[t] == k && w.hrows[t] < row)) {
            k = w.hkeys[t];
            row = w.hrows[t];
          }
        trows[t] = row;
      }
      if (trows[0] == UINT32_MAX) {   // no row has mass left
        filled = r;
        break;
      }
      for (uint32_t t = 0; t < L; t++) KMB_RET(fetch_row(trows[t], trial.data() + static_cast<size_t>(t) * D));
      for (size_t s = 0; s < devs.size(); s++) {
        Dev& d = devs[s];
        Work& w = wk[s];
        KMB_CU(cudaSetDevice(d.dev), kmcudaRuntimeError);
        KMB_CU(cudaMemcpyAsync(w.T.get(), trial.data(), sizeof(float) * trial.size(), cudaMemcpyHostToDevice, d.st),
               kmcudaMemoryCopyError);
        KMB_CU(cudaMemcpyAsync(w.rows.get(), trows.data(), sizeof(uint32_t) * L, cudaMemcpyHostToDevice, d.st),
               kmcudaMemoryCopyError);
        KMB_CU(launch_gpp_trial(metric, d.X, d.len, d.off, D, w.T, L, w.rows, d.dists, d.w.get(), w.ctl, w.dprime,
                                w.bsum, d.st), kmcudaRuntimeError);
        KMB_CU(launch_gpp_pick(w.bsum, d.len, L, w.ctl, w.rows, w.phis, false, nullptr, 0, D, nullptr, nullptr,
                               nullptr, d.st), kmcudaRuntimeError);
        KMB_CU(cudaMemcpyAsync(w.hphis.data(), w.phis.get(), sizeof(double) * L, cudaMemcpyDeviceToHost, d.st),
               kmcudaMemoryCopyError);
      }
      KMB_RET(sync_all());
      uint32_t best = 0;
      double best_phi = 0;
      for (uint32_t t = 0; t < L; t++) {
        double phi = 0;
        for (const Work& w : wk) phi += w.hphis[t];   // device order
        if (t == 0 || phi < best_phi) {
          best = t;
          best_phi = phi;
        }
      }
      rows[r] = trows[best];
      pots[r] = best_phi;
      memcpy(hostC.data() + static_cast<size_t>(r) * D, trial.data() + static_cast<size_t>(best) * D,
             sizeof(float) * D);
      const GppCtl next{best, trows[best], 0, 0};
      for (size_t s = 0; s < devs.size(); s++) {
        KMB_CU(cudaSetDevice(devs[s].dev), kmcudaRuntimeError);
        KMB_CU(cudaMemcpyAsync(wk[s].ctl.get(), &next, sizeof(GppCtl), cudaMemcpyHostToDevice, devs[s].st),
               kmcudaMemoryCopyError);
      }
    }
    KMB_RET(sync_all());
  }
  if (verbosity > 1)
    for (uint32_t r = 1; r < filled; r++)
      printf("greedy k-means++ round %" PRIu32 ": row %" PRIu32 ", potential %.17g\n", r, rows[r], pots[r]);
  for (auto& d : devs) d.dists.release();
  wk.clear();
  if (filled == K) {
    KMB_INFO("greedy k-means++: potential %.17g\n", pots[K - 1]);
    return single ? kmcudaSuccess : set_centroids_from_host(hostC.data());
  }
  KMB_INFO("greedy k-means++: potential 0 after %" PRIu32 " centroids, the rest from the random walk\n", filled);
  std::vector<char> taken(N, 0);
  for (uint32_t r = 0; r < filled; r++) taken[rows[r]] = 1;
  srand(seed);
  KMB_RET(fill_random(hostC.data(), filled, &taken, "greedy k-means++"));
  return set_centroids_from_host(hostC.data());
}

KMCUDAResult Job::init_centroids(KMCUDAInitMethod method, const void* init_params, uint32_t seed,
                                 int device_ptrs, bool fp16x2, const float* user_centroids) {
  if (metric == 1 && !fp16x2) {  // three probe samples must be unit length (kmcuda.cc:195-219)
    std::vector<float> row(D);
    for (uint32_t s : {0u, N / 2, N - 1}) {
      KMB_RET(fetch_row(s, row.data()));
      double norm = 0;
      for (int f = 0; f < D; f++) norm += row[f] * row[f];
      const float high = 1.00001, low = 0.99999;
      if (norm > high || norm < low) {
        KMB_INFO("error: angular distance: samples[%" PRIu32 "] has L2 norm = %f which is outside [%f, %f]\n",
                 s, norm, low, high);
        return kmcudaInvalidArguments;
      }
    }
  }
  srand(seed);
  switch (method) {
    case kmcudaInitMethodImport:   // (never borrowed: the run writes C)
      for (auto& d : devs) {
        KMB_CU(cudaSetDevice(d.dev), kmcudaRuntimeError);
        KMB_RET(copy_in(d.C, user_centroids, static_cast<size_t>(K) * D, d.dev, device_ptrs, fp16x2, d.st, verbosity,
                        false, false));
      }
      KMB_RET(sync_all());
      break;
    case kmcudaInitMethodRandom:
      KMB_RET(init_random());
      break;
    case kmcudaInitMethodPlusPlus:
      KMB_RET(init_plusplus());
      break;
    case kmcudaInitMethodAFKMC2: {
      uint32_t m = init_params ? *reinterpret_cast<const uint32_t*>(init_params) : 0;
      if (m == 0) {
        m = 200;
      } else if (m > N / 2) {
        KMB_INFO("afkmc2: m > %" PRIu32 " is not supported (got %" PRIu32 ")\n", N / 2, m);
        return kmcudaInvalidArguments;
      }
      KMB_RET(init_afkmc2(m, seed));
      break;
    }
    case kmcudaInitMethodKMeansParallel: {
      const uint32_t r = init_params ? *reinterpret_cast<const uint32_t*>(init_params) : 0;
      KMB_RET(init_kmeans_parallel(r ? r : kKMeansParallelRounds, seed));   // (r <= 32: kmeans_impl)
      break;
    }
    case kmcudaInitMethodGreedyPlusPlus: {
      const uint32_t t = init_params ? *reinterpret_cast<const uint32_t*>(init_params) : 0;
      KMB_RET(init_greedy_plusplus(t ? t : greedy_plusplus_trials(K), seed));   // (t <= 32: kmeans_impl)
      break;
    }
    default:
      return kmcudaInvalidArguments;
  }
  KMB_INFO("\rdone            \n");
  return kmcudaSuccess;
}
}  // namespace kmb
