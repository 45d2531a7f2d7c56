// Speaker gallery (dg_gallery_*): an enrolled gallery on the device and the standalone nearest-entry query.  A dg_multi with
// a gallery (dg_multi_set_gallery, api_multi.cu) runs the same kernels in its ticks.
#include <limits.h>
#include <math.h>
#include <string.h>

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

// One launch of the standalone search over queries X [Q][D] whose claim-group segments start at seg [n_seg + 1] (seg[0] = 0,
// seg[n_seg] = Q), query q in claim group grp[q]; Q * D <= INT_MAX (gallery_nearest's row offsets).
static int query_launch(dg_gallery* g, const double* queries_dev, int Q, const int32_t* grp, const std::vector<int>& seg,
                        const int32_t* claimed_dev, double threshold, int32_t* entry_dev, double* dist_dev, cudaStream_t st) {
  const int n_seg = (int)seg.size() - 1;
  if ((long long)Q * g->D > INT_MAX) {   // only a claim group of 32 rows of more than 67 million dimensions gets here
    set_error("dg_gallery_query: " + std::to_string(Q) + " rows of dimension " + std::to_string(g->D) +
              " in one claim group exceed 2^31 - 1 elements");
    return DG_EINVAL;
  }
  std::vector<int2> qd((size_t)Q);
  for (int q = 0; q < Q; q++) qd[q] = make_int2(q, grp[q]);
  // the one-group plan of the tick's grouped search; every table travels in one copy
  std::vector<GalGroup> groups(1, GalGroup{g->E.as<double>(), g->En.as<double>(), threshold, g->G, 0, 0, 0, Q, 0, n_seg, 0});
  std::vector<GalWork> work;
  const int splits = gallery_plan(groups, work), n_work = (int)work.size();
  const std::vector<int2> segs((size_t)n_seg, make_int2(0, 0));
  const int2 gq = make_int2(0, Q);
  const size_t o_seg = ((size_t)Q * 8 + 15) & ~(size_t)15, o_segs = (o_seg + seg.size() * 4 + 15) & ~(size_t)15,
               o_groups = (o_segs + (size_t)n_seg * 8 + 15) & ~(size_t)15, o_gq = o_groups + sizeof(GalGroup),
               o_work = o_gq + 16, bytes = o_work + (size_t)n_work * sizeof(GalWork);
  std::vector<unsigned char> in(bytes);
  memcpy(in.data(), qd.data(), (size_t)Q * 8);
  memcpy(in.data() + o_seg, seg.data(), seg.size() * 4);
  memcpy(in.data() + o_segs, segs.data(), (size_t)n_seg * 8);
  memcpy(in.data() + o_groups, groups.data(), sizeof(GalGroup));
  memcpy(in.data() + o_gq, &gq, 8);
  memcpy(in.data() + o_work, work.data(), (size_t)n_work * sizeof(GalWork));
  if (g->ws_in.ensure(bytes) || g->ws_d.ensure((size_t)splits * Q * 8) || g->ws_e.ensure((size_t)splits * Q * 4)) return DG_ECUDA;
  // a copy from pageable memory: staged before cudaMemcpyAsync returns
  DG_CUDA(cudaMemcpyAsync(g->ws_in.p, in.data(), bytes, cudaMemcpyHostToDevice, st));
  const unsigned char* din = g->ws_in.as<unsigned char>();
  const int2* d_qd = reinterpret_cast<const int2*>(din);
  const GalGroup* d_groups = reinterpret_cast<const GalGroup*>(din + o_groups);
  int rc;
  if ((rc = launch_gallery_nearest(d_groups, reinterpret_cast<const GalWork*>(din + o_work), n_work,
                                   reinterpret_cast<const int2*>(din + o_gq), g->Dp, queries_dev, g->D, d_qd, Q, claimed_dev,
                                   g->ws_d.as<double>(), g->ws_e.as<int>(), st)) ||
      (rc = launch_gallery_claim(g->ws_d.as<double>(), g->ws_e.as<int>(), Q, d_qd, reinterpret_cast<const int*>(din + o_seg),
                                 reinterpret_cast<const int2*>(din + o_segs), n_seg, d_groups, const_cast<int32_t*>(claimed_dev),
                                 entry_dev, dist_dev, nullptr, 0, nullptr, nullptr, nullptr, st)))
    return rc;
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
  }
  seg.push_back(Q);
  // one launch per run of whole segments of at most INT_MAX / D rows (gallery_nearest keeps 32-bit row offsets): a single
  // launch unless Q * D exceeds 2^31 - 1
  const int rows_max = (int)std::max<long long>(32, INT_MAX / g->D);
  for (size_t s0 = 0; s0 + 1 < seg.size();) {
    size_t s1 = s0 + 1;
    while (s1 + 1 < seg.size() && seg[s1 + 1] - seg[s0] <= rows_max) s1++;
    const int q0 = seg[s0], n = seg[s1] - q0;
    std::vector<int> local(seg.begin() + s0, seg.begin() + s1 + 1);
    for (int& o : local) o -= q0;
    int rc;
    if ((rc = query_launch(g, queries_dev + (size_t)q0 * g->D, n, grp.data() + q0, local, claimed_dev, threshold,
                           entry_dev + q0, dist_dev + q0, st)))
      return rc;
    s0 = s1;
  }
  return DG_OK;
}
