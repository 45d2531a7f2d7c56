// Device post-path (dg_post_*) and the hyper-parameter sweep (dg_sweep_*), which share the turn download.
#include <math.h>
#include <string.h>

#include <algorithm>
#include <cmath>
#include <memory>

#include "host.cuh"

static const int DG_POST_PREFIX = 16384;   // turns copied back together with the header (one D2H in the common case)

// Where the results of a post-path launch land in pinned memory: the header at `at`, the turn count in the 16 bytes after it,
// then the first DG_POST_PREFIX turns.  In front of `at`: dg_post's plan, or dg_sweep's error flags.
struct TurnOut {
  size_t at, header_bytes;
  size_t total() const { return at + header_bytes; }
  size_t prefix() const { return total() + 16; }
  size_t end() const { return prefix() + (size_t)DG_POST_PREFIX * 4; }
};

// After the stream `st` has been synchronised: hands the header and the turns of a TurnOut layout in `pin` to the caller; the
// turns beyond the prefix come from `turns_dev`.  `who` names the entry point in the error.
static int download_turns(const char* who, const unsigned char* pin, const TurnOut& lay, const uint32_t* turns_dev,
                          int32_t* header_host, uint32_t* turns_host, int turn_cap_host, int* n_turns, cudaStream_t st) {
  unsigned int total = 0;
  memcpy(&total, pin + lay.total(), 4);
  if (n_turns) *n_turns = (int)total;
  memcpy(header_host, pin + lay.at, lay.header_bytes);
  if ((long long)total > (long long)turn_cap_host) {
    set_error(std::string(who) + ": turn buffer too small (" + std::to_string(total) + " turns)");
    return DG_EINVAL;
  }
  const unsigned int pre = std::min<unsigned int>(total, (unsigned int)DG_POST_PREFIX);
  memcpy(turns_host, pin + lay.prefix(), (size_t)pre * 4);
  if (total > pre) {     // a second copy for what did not travel with the header
    DG_CUDA(cudaMemcpyAsync(turns_host + pre, turns_dev + pre, (size_t)(total - pre) * 4, cudaMemcpyDeviceToHost, st));
    DG_CUDA(cudaStreamSynchronize(st));
  }
  return DG_OK;
}

// pinned layout of a dg_post step over B chunks: plan [B][4 + nw], then header [B][4], turn count, turn prefix
static TurnOut post_out(const dg_post* h, int B) { return {(size_t)B * (4 + h->nw) * 4, (size_t)B * 16}; }

extern "C" int dg_post_create(int frames, int local_speakers, int max_speakers, int num_windows, const double* hamming_host,
                              double tau, int device, dg_post** out) {
  if (!out || !hamming_host || frames < 1 || frames > 1023 || local_speakers < 1 || max_speakers < 1 || max_speakers > 64 ||
      num_windows < 1 || num_windows > 256) {
    set_error("dg_post_create: need 1 <= frames <= 1023, 1 <= max_speakers <= 64, 1 <= num_windows <= 256");
    return DG_EINVAL;
  }
  DG_CUDA(cudaSetDevice(device));
  std::unique_ptr<dg_post> h(new dg_post());
  h->device = device; h->F = frames; h->K = local_speakers; h->M = max_speakers; h->nw = num_windows; h->tau = tau;
  if (h->hamming.ensure((size_t)frames * 8) || h->total.ensure(16)) return DG_ECUDA;
  DG_CUDA(cudaMemcpy(h->hamming.p, hamming_host, (size_t)frames * 8, cudaMemcpyHostToDevice));
  const size_t hs = (size_t)std::max(1, num_windows - 1);
  for (int i = 0; i < 2; i++)
    if (h->hist_seg[i].ensure(hs * frames * local_speakers * 4) || h->hist_map[i].ensure(hs * local_speakers * 4)) return DG_ECUDA;
  *out = h.release();
  return DG_OK;
}

extern "C" int dg_post_reset(dg_post* h) {
  if (!h) return DG_EINVAL;
  h->n_hist = 0;
  return DG_OK;
}

extern "C" int dg_post_destroy(dg_post* h) {
  delete h;
  return DG_OK;
}

static int post_ensure(dg_post* h, int B) {
  if (B <= h->cap_B) return 0;
  const int stride = 4 + h->nw;
  // worst case: every second frame of every speaker starts a turn
  h->turn_cap = B * h->M * ((h->F + 1) / 2);
  if (h->plan.ensure((size_t)B * stride * 4) || h->header.ensure((size_t)B * 16 + 16) ||
      h->turns.ensure((size_t)h->turn_cap * 4))
    return DG_ECUDA;
  if (h->pin.ensure(post_out(h, B).end())) return DG_ECUDA;
  h->cap_B = B;
  return 0;
}

// enqueues plan upload, aggregation + binarisation + run-length kernel, history update and the D2H of the results on `st`
int post_enqueue(dg_post* h, const float* seg_dev, const int32_t* map_dev, int B, const int32_t* plan_host,
                 cudaStream_t st) {
  int rc;
  if ((rc = post_ensure(h, B))) return rc;
  const int stride = 4 + h->nw;
  unsigned char* pin = h->pin.as<unsigned char>();
  const size_t plan_bytes = (size_t)B * stride * 4;
  memcpy(pin, plan_host, plan_bytes);
  DG_CUDA(cudaMemcpyAsync(h->plan.p, pin, plan_bytes, cudaMemcpyHostToDevice, st));
  DG_CUDA(cudaMemsetAsync(h->total.p, 0, 4, st));
  if ((rc = launch_post(seg_dev, map_dev, h->hist_seg[h->cur].as<float>(), h->hist_map[h->cur].as<int32_t>(), h->n_hist, B,
                        h->F, h->K, h->M, h->nw, h->plan.as<int32_t>(), stride, h->hamming.as<double>(), h->tau,
                        h->header.as<int32_t>(), h->turns.as<uint32_t>(), h->turn_cap, h->total.as<unsigned int>(), st)))
    return rc;
  const int keep = std::min(h->nw - 1, h->n_hist + B);
  if (keep > 0) {
    if ((rc = launch_post_history(seg_dev, map_dev, h->hist_seg[h->cur].as<float>(), h->hist_map[h->cur].as<int32_t>(),
                                  h->n_hist, B, h->F, h->K, keep, h->hist_seg[h->cur ^ 1].as<float>(),
                                  h->hist_map[h->cur ^ 1].as<int32_t>(), st)))
      return rc;
    h->cur ^= 1;
  }
  h->n_hist = keep;
  const TurnOut lay = post_out(h, B);
  DG_CUDA(cudaMemcpyAsync(pin + lay.at, h->header.p, lay.header_bytes, cudaMemcpyDeviceToHost, st));
  DG_CUDA(cudaMemcpyAsync(pin + lay.total(), h->total.p, 4, cudaMemcpyDeviceToHost, st));
  DG_CUDA(cudaMemcpyAsync(pin + lay.prefix(), h->turns.p, (size_t)std::min(DG_POST_PREFIX, h->turn_cap) * 4,
                          cudaMemcpyDeviceToHost, st));
  return 0;
}

// after `st` has been synchronised: hands the results to the caller
int post_finish(dg_post* h, int B, int32_t* header_host, uint32_t* turns_host, int turn_cap_host, int* n_turns,
                cudaStream_t st) {
  return download_turns("dg_post_step", h->pin.as<unsigned char>(), post_out(h, B), h->turns.as<uint32_t>(), header_host,
                        turns_host, turn_cap_host, n_turns, st);
}

extern "C" int dg_post_step(dg_post* h, const float* seg_dev, const int32_t* map_dev, int B, const int32_t* plan_host,
                            int32_t* header_host, uint32_t* turns_host, int turn_cap_host, int* n_turns, void* stream) {
  if (!h || !seg_dev || !map_dev || !plan_host || !header_host || !turns_host || B < 1) {
    set_error("dg_post_step: bad arguments");
    return DG_EINVAL;
  }
  DG_CUDA(cudaSetDevice(h->device));
  cudaStream_t st = (cudaStream_t)stream;
  int rc;
  if ((rc = post_enqueue(h, seg_dev, map_dev, B, plan_host, st))) return rc;
  DG_CUDA(cudaStreamSynchronize(st));
  return post_finish(h, B, header_host, turns_host, turn_cap_host, n_turns, st);
}

// ============================================================================= hyper-parameter sweep
// T independent clustering + post-path states over ONE set of network outputs (seg, emb of a whole file): the reference tunes
// tau_active, rho_update and delta_new by re-running its whole pipeline per trial (Optimizer.objective -> Benchmark), although
// none of the three reaches the networks.  Clustering: one CTA per state (cluster.cu); post-path: one CTA per (chunk, state)
// over all chunks at once, without history (post.cu).
struct dg_sweep {
  int device = 0, M = 0, D = 0, F = 0, K = 0, nw = 1;
  DevBuf hamming, in, centers, active, init, prep, prep_d, maps, header, turns, total;
  DevBuf score_in, hoff, hseg, comp;   // dg_sweep_score: chunk times and reference, hypothesis segments, components
  PinnedBuf pin;                  // params, taus and plan in; error flags, header, total and a turn prefix out
};

extern "C" int dg_sweep_create(int max_speakers, int dim, int frames, int local_speakers, int num_windows,
                               const double* hamming_host, int device, dg_sweep** out) {
  if (!out || !hamming_host || max_speakers < 1 || max_speakers > 32 || dim < 1 || local_speakers < 1 || local_speakers > 8 ||
      local_speakers > max_speakers || frames < 1 || frames > 1023 || num_windows < 1 || num_windows > 256) {
    set_error("dg_sweep_create: need 1 <= max_speakers <= 32, dim >= 1, 1 <= local_speakers <= min(8, max_speakers), "
              "1 <= frames <= 1023, 1 <= num_windows <= 256");
    return DG_EINVAL;
  }
  DG_CUDA(cudaSetDevice(device));
  std::unique_ptr<dg_sweep> h(new dg_sweep());
  h->device = device; h->M = max_speakers; h->D = dim; h->F = frames; h->K = local_speakers; h->nw = num_windows;
  if (h->hamming.ensure((size_t)frames * 8) || h->total.ensure(16)) return DG_ECUDA;
  DG_CUDA(cudaMemcpy(h->hamming.p, hamming_host, (size_t)frames * 8, cudaMemcpyHostToDevice));
  *out = h.release();
  return DG_OK;
}

extern "C" int dg_sweep_destroy(dg_sweep* h) {
  delete h;
  return DG_OK;
}

// the argument checks dg_sweep_run and dg_sweep_score share (before any launch)
static int sweep_check(const char* who, dg_sweep* h, const float* seg_dev, const float* emb_dev, int N,
                       const double* params_host, int T, const int32_t* plan_host) {
  if (!h || !seg_dev || !emb_dev || !params_host || !plan_host || N < 1 || T < 1 || T > 65535) {
    set_error(std::string(who) + ": bad arguments (need N >= 1, 1 <= T <= 65535, non-null buffers)");
    return DG_EINVAL;
  }
  for (int i = 0; i < 3 * T; i++)
    if (!std::isfinite(params_host[i])) {
      set_error(std::string(who) + ": trial " + std::to_string(i / 3) + " has a parameter that is not finite");
      return DG_EINVAL;
    }
  return DG_OK;
}

// pinned output layout of sweep_cluster_post: error flags [T][2], then header [T][N][4], turn count, turn prefix
static TurnOut sweep_out(int T, int N) { return {(size_t)T * 8, (size_t)T * N * 16}; }

// Clustering + post-path of T trials over the N chunks: header [T][N][4] and turns stay on the device (h->header, h->turns),
// the turn count comes back in *total.  with_header: the header and a prefix of the turns travel to the pinned buffer in the
// same copy as the count (sweep_out layout).  Synchronises `st`.
static int sweep_cluster_post(dg_sweep* h, const float* seg_dev, const float* emb_dev, int N, const double* params_host,
                              int T, const int32_t* plan_host, int32_t* maps_dev, double* centers_dev, bool with_header,
                              cudaStream_t st, unsigned int* total_out) {
  const int stride = 4 + h->nw, M = h->M, D = h->D, K = h->K, F = h->F;
  // host -> device: params [T][3], taus [T], plan [N][stride], one copy
  const size_t params_b = (size_t)T * 24, taus_b = (size_t)T * 8, plan_b = (size_t)N * stride * 4;
  const size_t in_b = params_b + taus_b + plan_b;
  const TurnOut lay = sweep_out(T, N);
  const size_t init_b = lay.at, header_b = lay.header_bytes;
  // the device turn buffer starts at a guess and grows to the true count (the kernel counts every turn, writes those that fit)
  const size_t turn_guess = std::max<size_t>((size_t)T * N * 8, (size_t)DG_POST_PREFIX);
  if (h->in.ensure(in_b) || h->centers.ensure((size_t)T * M * D * 8) || h->active.ensure((size_t)T * 32 * 4) ||
      h->init.ensure(init_b) || h->prep.ensure(cluster_prep_floats(N, K) * 4 + 16) ||
      h->prep_d.ensure(cluster_prep_doubles(N, K) * 8 + 16) || (!maps_dev && h->maps.ensure((size_t)T * N * K * 4)) ||
      h->header.ensure(header_b) || h->turns.ensure(turn_guess * 4) || h->pin.ensure(std::max(in_b, lay.end())))
    return DG_ECUDA;
  unsigned char* pin = h->pin.as<unsigned char>();
  double* p_taus = reinterpret_cast<double*>(pin + params_b);
  memcpy(pin, params_host, params_b);
  for (int t = 0; t < T; t++) p_taus[t] = params_host[3 * t];
  memcpy(pin + params_b + taus_b, plan_host, plan_b);
  unsigned char* din = h->in.as<unsigned char>();
  DG_CUDA(cudaMemcpyAsync(din, pin, in_b, cudaMemcpyHostToDevice, st));
  const double* d_params = reinterpret_cast<const double*>(din);
  const double* d_taus = reinterpret_cast<const double*>(din + params_b);
  const int32_t* d_plan = reinterpret_cast<const int32_t*>(din + params_b + taus_b);
  int32_t* maps = maps_dev ? maps_dev : h->maps.as<int32_t>();
  // every state starts empty (reference: a new OnlineSpeakerClustering per trial)
  DG_CUDA(cudaMemsetAsync(h->centers.p, 0, (size_t)T * M * D * 8, st));
  DG_CUDA(cudaMemsetAsync(h->active.p, 0, (size_t)T * 32 * 4, st));
  DG_CUDA(cudaMemsetAsync(h->init.p, 0, init_b, st));
  ClusterParams p{};
  p.M = M;
  p.D = D;
  p.metric = 0;
  int rc;
  if ((rc = launch_cluster_sweep(p, d_params, T, seg_dev, emb_dev, N, F, K, h->centers.as<double>(), h->active.as<int>(),
                                 h->init.as<int>(), h->prep.as<float>(), h->prep_d.as<double>(), maps, st)))
    return rc;
  if (centers_dev)
    DG_CUDA(cudaMemcpyAsync(centers_dev, h->centers.p, (size_t)T * M * D * 8, cudaMemcpyDeviceToDevice, st));
  unsigned int total = 0;
  for (int attempt = 0; attempt < 2; attempt++) {
    const int cap = (int)std::min<size_t>(h->turns.bytes / 4, (size_t)INT32_MAX);
    DG_CUDA(cudaMemsetAsync(h->total.p, 0, 4, st));
    if ((rc = launch_post(seg_dev, maps, nullptr, nullptr, 0, N, F, K, M, h->nw, d_plan, stride, h->hamming.as<double>(), 0.0,
                          h->header.as<int32_t>(), h->turns.as<uint32_t>(), cap, h->total.as<unsigned int>(), st, d_taus, T)))
      return rc;
    DG_CUDA(cudaMemcpyAsync(pin, h->init.p, init_b, cudaMemcpyDeviceToHost, st));
    if (with_header) DG_CUDA(cudaMemcpyAsync(pin + lay.at, h->header.p, header_b, cudaMemcpyDeviceToHost, st));
    DG_CUDA(cudaMemcpyAsync(pin + lay.total(), h->total.p, 4, cudaMemcpyDeviceToHost, st));
    if (with_header)
      DG_CUDA(cudaMemcpyAsync(pin + lay.prefix(), h->turns.p, (size_t)std::min(DG_POST_PREFIX, cap) * 4,
                              cudaMemcpyDeviceToHost, st));
    DG_CUDA(cudaStreamSynchronize(st));
    memcpy(&total, pin + lay.total(), 4);
    if (total <= (unsigned int)cap) break;
    // more turns than the device buffer holds: grow it to the count and binarise again (the maps are unchanged)
    if (h->turns.ensure((size_t)total * 4)) return DG_ECUDA;
  }
  const int32_t* flags = reinterpret_cast<const int32_t*>(pin);
  for (int t = 0; t < T; t++)
    if (flags[2 * t + 1]) {
      set_error("Cannot update unknown centers");   // reference clustering.py:98 (AssertionError)
      return DG_EINVAL;
    }
  *total_out = total;
  return DG_OK;
}

extern "C" int dg_sweep_run(dg_sweep* h, const float* seg_dev, const float* emb_dev, int N, const double* params_host, int T,
                            const int32_t* plan_host, int32_t* maps_dev, double* centers_dev, int32_t* header_host,
                            uint32_t* turns_host, int turn_cap_host, int* n_turns, void* stream) {
  if (!header_host || !turns_host) {
    set_error("dg_sweep_run: bad arguments (need N >= 1, 1 <= T <= 65535, non-null buffers)");
    return DG_EINVAL;
  }
  int rc;
  if ((rc = sweep_check("dg_sweep_run", h, seg_dev, emb_dev, N, params_host, T, plan_host))) return rc;
  DG_CUDA(cudaSetDevice(h->device));
  cudaStream_t st = (cudaStream_t)stream;
  unsigned int total = 0;
  if ((rc = sweep_cluster_post(h, seg_dev, emb_dev, N, params_host, T, plan_host, maps_dev, centers_dev, true, st, &total)))
    return rc;
  return download_turns("dg_sweep_run", h->pin.as<unsigned char>(), sweep_out(T, N), h->turns.as<uint32_t>(), header_host,
                        turns_host, turn_cap_host, n_turns, st);
}

// the reference rows: finite, start < end, labels in [0, R), each label's rows in time order without overlap
static int sweep_check_reference(const double* ref_host, const int32_t* ref_label_host, int S, int R) {
  if (R < 0 || R > 32 || S < 0 || (S > 0 && (!ref_host || !ref_label_host))) {
    set_error("dg_sweep_score: need 0 <= reference labels <= 32, rows >= 0, non-null reference arrays");
    return DG_EINVAL;
  }
  double last[32];
  for (int r = 0; r < 32; r++) last[r] = -INFINITY;
  for (int i = 0; i < S; i++) {
    const double a = ref_host[2 * i], b = ref_host[2 * i + 1];
    const int r = ref_label_host[i];
    if (r < 0 || r >= R) {
      set_error("dg_sweep_score: reference row " + std::to_string(i) + " has a label outside [0, R)");
      return DG_EINVAL;
    }
    if (!std::isfinite(a) || !std::isfinite(b) || !(a < b)) {
      set_error("dg_sweep_score: reference row " + std::to_string(i) + " is not finite, empty or reversed");
      return DG_EINVAL;
    }
    if (a < last[r]) {
      set_error("dg_sweep_score: reference row " + std::to_string(i) + " is out of order or overlaps an earlier row of its label");
      return DG_EINVAL;
    }
    last[r] = b;
  }
  return DG_OK;
}

extern "C" int dg_sweep_score(dg_sweep* h, const float* seg_dev, const float* emb_dev, int N, const double* params_host,
                              int T, const int32_t* plan_host, const double* out_start_host, const double* out_res_host,
                              double shift, double collar, const double* ref_host, const int32_t* ref_label_host, int S,
                              int R, double* components_host, int32_t* hyp_offsets_dev, double* hyp_segments_dev,
                              int hyp_cap, void* stream) {
  int rc;
  if ((rc = sweep_check("dg_sweep_score", h, seg_dev, emb_dev, N, params_host, T, plan_host))) return rc;
  if (!out_start_host || !out_res_host || !components_host || hyp_cap < 0 || !std::isfinite(shift) ||
      !std::isfinite(collar) || collar < 0) {
    set_error("dg_sweep_score: bad arguments (need chunk times, a components buffer, finite shift, finite collar >= 0, "
              "hyp_cap >= 0)");
    return DG_EINVAL;
  }
  for (int c = 0; c < N; c++)
    if (!std::isfinite(out_start_host[c]) || !std::isfinite(out_res_host[c])) {
      set_error("dg_sweep_score: chunk " + std::to_string(c) + " has an output time that is not finite");
      return DG_EINVAL;
    }
  if ((rc = sweep_check_reference(ref_host, ref_label_host, S, R))) return rc;
  DG_CUDA(cudaSetDevice(h->device));
  cudaStream_t st = (cudaStream_t)stream;
  unsigned int total = 0;
  if ((rc = sweep_cluster_post(h, seg_dev, emb_dev, N, params_host, T, plan_host, nullptr, nullptr, false, st, &total)))
    return rc;
  const int M = h->M, TM = T * M;
  // host -> device, one copy: out_start [N], out_res [N], reference segments [S][2] grouped by label, label offsets [R + 1]
  const size_t times_b = (size_t)N * 16, rseg_b = (size_t)S * 16, roff_b = (size_t)(R + 1) * 4;
  const size_t in_b = times_b + rseg_b + roff_b, comp_b = (size_t)T * 40;
  if (h->score_in.ensure(in_b) || h->hoff.ensure((size_t)(TM + 1) * 4) || h->hseg.ensure((size_t)std::max(total, 1u) * 16) ||
      h->comp.ensure(comp_b) || h->pin.ensure(std::max(in_b, comp_b + 16)))
    return DG_ECUDA;
  unsigned char* pin = h->pin.as<unsigned char>();
  memcpy(pin, out_start_host, (size_t)N * 8);
  memcpy(pin + (size_t)N * 8, out_res_host, (size_t)N * 8);
  double* rseg = reinterpret_cast<double*>(pin + times_b);
  int32_t* roff = reinterpret_cast<int32_t*>(pin + times_b + rseg_b);
  for (int r = 0; r <= R; r++) roff[r] = 0;
  for (int i = 0; i < S; i++) roff[ref_label_host[i] + 1]++;
  for (int r = 0; r < R; r++) roff[r + 1] += roff[r];
  int fill[32];
  for (int r = 0; r < R; r++) fill[r] = roff[r];
  for (int i = 0; i < S; i++) {     // stable: each label keeps its rows' order
    const int o = fill[ref_label_host[i]]++;
    rseg[2 * o] = ref_host[2 * i];
    rseg[2 * o + 1] = ref_host[2 * i + 1];
  }
  unsigned char* din = h->score_in.as<unsigned char>();
  DG_CUDA(cudaMemcpyAsync(din, pin, in_b, cudaMemcpyHostToDevice, st));
  const double* d_start = reinterpret_cast<const double*>(din);
  const double* d_res = d_start + N;
  const double* d_rseg = reinterpret_cast<const double*>(din + times_b);
  const int* d_roff = reinterpret_cast<const int*>(din + times_b + rseg_b);
  int* hoff = h->hoff.as<int>();
  if ((rc = launch_der_hyp_count(h->header.as<int32_t>(), h->turns.as<uint32_t>(), T, N, M, d_start, d_res, shift, collar,
                                 hoff, st)) ||
      (rc = launch_der_hyp_write(h->header.as<int32_t>(), h->turns.as<uint32_t>(), T, N, M, d_start, d_res, shift, collar,
                                 hoff, h->hseg.as<double>(), hyp_segments_dev, hyp_cap, st)) ||
      (rc = launch_der_score(hoff, h->hseg.as<double>(), T, M, d_roff, d_rseg, R, h->comp.as<double>(), st)))
    return rc;
  if (hyp_offsets_dev) DG_CUDA(cudaMemcpyAsync(hyp_offsets_dev, hoff, (size_t)(TM + 1) * 4, cudaMemcpyDeviceToDevice, st));
  DG_CUDA(cudaMemcpyAsync(pin, h->comp.p, comp_b, cudaMemcpyDeviceToHost, st));
  DG_CUDA(cudaMemcpyAsync(pin + comp_b, hoff + TM, 4, cudaMemcpyDeviceToHost, st));
  DG_CUDA(cudaStreamSynchronize(st));
  memcpy(components_host, pin, comp_b);
  int n_seg = 0;
  memcpy(&n_seg, pin + comp_b, 4);
  if (hyp_segments_dev && n_seg > hyp_cap) {
    set_error("dg_sweep_score: hypothesis segment buffer too small (" + std::to_string(n_seg) + " segments)");
    return DG_EINVAL;
  }
  return DG_OK;
}
