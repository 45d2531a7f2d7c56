// Speaker gallery (dg_gallery_*): an enrolled gallery on the device and the standalone nearest-entry query.  A dg_multi with
// a gallery (dg_multi_set_gallery, api_multi.cu) runs the same kernels in its ticks.
#include <math.h>

#include <algorithm>
#include <cmath>
#include <memory>
#include <vector>

#include "host.cuh"

static bool threshold_ok(double t) { return std::isfinite(t) && t > 0.0 && t <= 2.0; }

extern "C" int dg_gallery_create(const double* centroids_host, int G, int D, int device, dg_gallery** out) {
  const char* who = "dg_gallery_create";
  if (!centroids_host || !out) {
    set_error(std::string(who) + ": null table or output");
    return DG_EINVAL;
  }
  if (G < 1 || G > (1 << 20) || D < 2 || D % 2) {
    set_error(std::string(who) + ": need 1 <= G <= 1048576 entries of an even dimension D >= 2, got G = " + std::to_string(G) +
              ", D = " + std::to_string(D));
    return DG_EINVAL;
  }
  for (int i = 0; i < G; i++) {
    double ss = 0.0;
    bool finite = true;
    for (int d = 0; d < D; d++) {
      const double x = centroids_host[(size_t)i * D + d];
      finite = finite && std::isfinite(x);
      ss += x * x;
    }
    if (!finite || !(ss > 0.0)) {
      set_error(std::string(who) + ": entry " + std::to_string(i) + (finite ? " has a zero norm" : " is not finite"));
      return DG_EINVAL;
    }
  }
  DG_CUDA(cudaSetDevice(device));
  std::unique_ptr<dg_gallery> g(new dg_gallery());
  g->device = device;
  g->G = G;
  g->D = D;
  g->Gp = (G + GAL_TILE_E - 1) / GAL_TILE_E * GAL_TILE_E;
  g->Dp = (D + GAL_KC - 1) / GAL_KC * GAL_KC;
  if (g->E.ensure((size_t)g->Gp * g->Dp * 8) || g->En.ensure((size_t)G * 8)) return DG_ECUDA;   // zeroed
  DG_CUDA(cudaMemcpy2D(g->E.p, (size_t)g->Dp * 8, centroids_host, (size_t)D * 8, (size_t)D * 8, G, cudaMemcpyHostToDevice));
  int rc;
  if ((rc = launch_gallery_norms(g->E.as<double>(), G, g->Dp, g->En.as<double>(), 0))) return rc;
  DG_CUDA(cudaDeviceSynchronize());
  *out = g.release();
  return DG_OK;
}

extern "C" int dg_gallery_destroy(dg_gallery* g) {
  delete g;
  return DG_OK;
}

extern "C" int dg_gallery_query(dg_gallery* g, const double* queries_dev, int Q, const int32_t* group_dev,
                                const int32_t* claimed_dev, double threshold, int32_t* entry_dev, double* dist_dev, void* stream) {
  const char* who = "dg_gallery_query";
  if (!g || !queries_dev || Q < 1 || !group_dev || !entry_dev || !dist_dev) {
    set_error(std::string(who) + ": need a gallery, Q >= 1 queries and non-null groups and outputs");
    return DG_EINVAL;
  }
  if (!threshold_ok(threshold)) {
    set_error(std::string(who) + ": need a finite threshold in (0, 2]");
    return DG_EINVAL;
  }
  DG_CUDA(cudaSetDevice(g->device));
  cudaStream_t st = (cudaStream_t)stream;
  std::vector<int32_t> grp((size_t)Q);
  DG_CUDA(cudaMemcpyAsync(grp.data(), group_dev, (size_t)Q * 4, cudaMemcpyDeviceToHost, st));
  DG_CUDA(cudaStreamSynchronize(st));
  // the segments: each group one contiguous run of at most 32 queries
  std::vector<int2> qd((size_t)Q);
  std::vector<int> seg(1, 0);
  std::vector<char> seen;
  for (int q = 0; q < Q; q++) {
    const int r = grp[q];
    if (r < 0) {
      set_error(std::string(who) + ": query " + std::to_string(q) + " has a negative group");
      return DG_EINVAL;
    }
    if (q > 0 && r != grp[q - 1]) seg.push_back(q);
    if (q == 0 || r != grp[q - 1]) {
      if ((size_t)r >= seen.size()) seen.resize((size_t)r + 1, 0);
      if (seen[r]) {
        set_error(std::string(who) + ": the queries of group " + std::to_string(r) + " are not one contiguous run");
        return DG_EINVAL;
      }
      seen[r] = 1;
    }
    if (q - seg.back() >= 32) {
      set_error(std::string(who) + ": group " + std::to_string(r) + " has more than 32 queries");
      return DG_EINVAL;
    }
    qd[q] = make_int2(q, r);
  }
  seg.push_back(Q);
  const int n_seg = (int)seg.size() - 1, splits = gallery_splits(g->G, Q);
  if (g->ws_q.ensure((size_t)Q * 8) || g->ws_seg.ensure(seg.size() * 4) || g->ws_d.ensure((size_t)splits * Q * 8) ||
      g->ws_e.ensure((size_t)splits * Q * 4))
    return DG_ECUDA;
  // copies from pageable memory: staged before cudaMemcpyAsync returns
  DG_CUDA(cudaMemcpyAsync(g->ws_q.p, qd.data(), (size_t)Q * 8, cudaMemcpyHostToDevice, st));
  DG_CUDA(cudaMemcpyAsync(g->ws_seg.p, seg.data(), seg.size() * 4, cudaMemcpyHostToDevice, st));
  int rc;
  if ((rc = launch_gallery_nearest(g->E.as<double>(), g->En.as<double>(), g->G, g->Gp, g->Dp, queries_dev, g->D,
                                   g->ws_q.as<int2>(), nullptr, Q, claimed_dev, splits, g->ws_d.as<double>(), g->ws_e.as<int>(),
                                   st)) ||
      (rc = launch_gallery_claim(g->ws_d.as<double>(), g->ws_e.as<int>(), splits, Q, g->ws_q.as<int2>(), g->ws_seg.as<int>(),
                                 n_seg, threshold, const_cast<int32_t*>(claimed_dev), entry_dev, dist_dev, nullptr, 0, nullptr,
                                 nullptr, nullptr, st)))
    return rc;
  return DG_OK;
}
