// Device post-path (dg_post_*), the hyper-parameter sweep (dg_sweep_*) and the voice activity detection sweep (dg_vad_sweep_*),
// which share the turn download; the two sweeps share the DER scoring sequence (der_components).
#include <math.h>
#include <string.h>

#include <algorithm>
#include <cmath>
#include <memory>

#include "host.cuh"

int download_turns(const char* who, const unsigned char* pin, const TurnOut& lay, const uint32_t* turns_dev,
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

// ============================================================================= plan rows
int check_plan_row(const char* who, const int32_t* pl, int row, int nw, int before, int F) {
  const int nb = pl[0], nf = pl[1], nfo = pl[2] > 0 ? pl[2] : nf;
  if (nb < 1 || nb > nw || nb - 1 > before || nf < 1 || pl[2] < 0 || nfo > std::min(F + 1, 1023)) {
    set_error(std::string(who) + ": plan row " + std::to_string(row) + " is not a plan of its stream or file (buffers " +
              std::to_string(nb) + ", frames " + std::to_string(nfo) + ")");
    return DG_EINVAL;
  }
  return DG_OK;
}

// the plan rows of N chunks in nf files (chunk_off [nf + 1], checked), each file a fresh stream
static int check_file_plans(const char* who, const int32_t* plan, int nf, const int32_t* chunk_off, int nw, int F) {
  int rc;
  for (int f = 0; f < nf; f++)
    for (int c = chunk_off[f]; c < chunk_off[f + 1]; c++)
      if ((rc = check_plan_row(who, plan + (size_t)c * (4 + nw), c, nw, c - chunk_off[f], F))) return rc;
  return DG_OK;
}

int post_check(const char* who, const dg_post* h, int B, const int32_t* plan_host) {
  int rc;
  for (int c = 0; c < B; c++)
    if ((rc = check_plan_row(who, plan_host + (size_t)c * (4 + h->nw), c, h->nw, h->n_hist + c, h->F))) return rc;
  return DG_OK;
}

// ============================================================================= device post-path of one stream
// A dg_post step is one stream in slot 0 of post_slots_kernel.  Pinned layout over B chunks: what travels to h->in in one
// copy -- {tau, 0, 0} float64, the stream's TickSlot, rows [B] {0, c}, plan [B][4 + nw] -- then header [B][4], turn count,
// turn prefix
static const size_t POST_ROWS_AT = 24 + sizeof(TickSlot);
static size_t post_in_bytes(const dg_post* h, int B) { return POST_ROWS_AT + (size_t)B * 8 + (size_t)B * (4 + h->nw) * 4; }
static TurnOut post_out(const dg_post* h, int B) { return {post_in_bytes(h, B), (size_t)B * 16}; }

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
  if (h->hist_seg.ensure(2 * hs * frames * local_speakers * 4) || h->hist_map.ensure(2 * hs * local_speakers * 4))
    return DG_ECUDA;
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
  h->turn_cap = post_turn_cap(B, h->M, h->F);
  if (h->in.ensure(post_in_bytes(h, B)) || h->header.ensure((size_t)B * 16 + 16) || h->turns.ensure((size_t)h->turn_cap * 4))
    return DG_ECUDA;
  if (h->pin.ensure(post_out(h, B).end())) return DG_ECUDA;
  h->cap_B = B;
  return 0;
}

// enqueues the upload, aggregation + binarisation + run-length kernel, history update and the D2H of the results on `st`
// (plan rows checked by post_check)
int post_enqueue(dg_post* h, const float* seg_dev, const int32_t* map_dev, int B, const int32_t* plan_host,
                 cudaStream_t st) {
  int rc;
  if ((rc = post_ensure(h, B))) return rc;
  const int stride = 4 + h->nw;
  const size_t plan_at = POST_ROWS_AT + (size_t)B * 8;
  unsigned char* pin = h->pin.as<unsigned char>();
  const double params[3] = {h->tau, 0.0, 0.0};
  const TickSlot ts{0, 0, B, h->cur, h->n_hist, h->nw, {0, 0}};
  memcpy(pin, params, 24);
  memcpy(pin + 24, &ts, sizeof ts);
  int2* rows = reinterpret_cast<int2*>(pin + POST_ROWS_AT);
  for (int c = 0; c < B; c++) rows[c] = make_int2(0, c);
  memcpy(pin + plan_at, plan_host, (size_t)B * stride * 4);
  unsigned char* din = h->in.as<unsigned char>();
  DG_CUDA(cudaMemcpyAsync(din, pin, post_in_bytes(h, B), cudaMemcpyHostToDevice, st));
  DG_CUDA(cudaMemsetAsync(h->total.p, 0, 4, st));
  const TickSlot* d_ts = reinterpret_cast<const TickSlot*>(din + 24);
  if ((rc = launch_post_slots(seg_dev, map_dev, h->hist_seg.as<float>(), h->hist_map.as<int32_t>(), d_ts,
                              reinterpret_cast<const int2*>(din + POST_ROWS_AT), 1, B, h->F, h->K, h->M, h->nw,
                              reinterpret_cast<const int32_t*>(din + plan_at), stride, h->hamming.as<double>(),
                              reinterpret_cast<const double*>(din), h->header.as<int32_t>(), h->turns.as<uint32_t>(),
                              h->turn_cap, h->total.as<unsigned int>(), st)) ||
      (rc = launch_post_slots_history(seg_dev, map_dev, h->hist_seg.as<float>(), h->hist_map.as<int32_t>(), d_ts, 1, 1, h->F,
                                      h->K, h->nw, st)))
    return rc;
  if (h->nw > 1) {
    h->n_hist = std::min(h->nw - 1, h->n_hist + B);
    h->cur ^= 1;
  }
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
  int rc;
  if ((rc = post_check("dg_post_step", h, B, plan_host))) return rc;
  DG_CUDA(cudaSetDevice(h->device));
  cudaStream_t st = (cudaStream_t)stream;
  if ((rc = post_enqueue(h, seg_dev, map_dev, B, plan_host, st))) return rc;
  DG_CUDA(cudaStreamSynchronize(st));
  return post_finish(h, B, header_host, turns_host, turn_cap_host, n_turns, st);
}

// ============================================================================= hyper-parameter sweep
// T independent clustering + post-path states over ONE set of network outputs (seg, emb of a whole file): the reference tunes
// tau_active, rho_update and delta_new by re-running its whole pipeline per trial (Optimizer.objective -> Benchmark), although
// none of the three reaches the networks.  Clustering: one CTA per state (cluster.cu); post-path: one CTA per (chunk, state)
// over all chunks at once, without history (post.cu).

// the device buffers of der_components: chunk times and reference in, hypothesis offsets and segments, components out
struct DerBufs {
  DevBuf in, hoff, hseg, comp;
};

// The scored pieces of every file a scoring call covers (dg_sweep_set_scored_regions / dg_vad_sweep_set_scored_regions): file
// f's pieces are rows [off[f], off[f + 1]), sorted, apart by more than 1e-6 s, finite and each truthy.  nf = 0: none, the
// hypotheses are scored whole.
struct ScoredRegions {
  int nf = 0;
  std::vector<double> rows;    // [S][2]
  std::vector<int32_t> off;    // [nf + 1]
};

// the arguments are checked before the handle, so that the checks run without a device; r: the handle's regions
static int set_scored_regions(const char* who, ScoredRegions* r, int nf, const double* rows, const int32_t* off) {
  if (nf < 0 || (nf > 0 && !off)) {
    set_error(std::string(who) + ": bad arguments (need num_files >= 0 and row offsets when num_files > 0)");
    return DG_EINVAL;
  }
  if (nf > 0 && off[0] != 0) {
    set_error(std::string(who) + ": scored region offsets must start at 0");
    return DG_EINVAL;
  }
  for (int f = 0; f < nf; f++)
    if (off[f + 1] < off[f]) {
      set_error(std::string(who) + ": scored region offsets of file " + std::to_string(f) + " decrease");
      return DG_EINVAL;
    }
  const int S = nf > 0 ? off[nf] : 0;
  if (S > 0 && !rows) {
    set_error(std::string(who) + ": non-null rows needed for " + std::to_string(S) + " scored regions");
    return DG_EINVAL;
  }
  for (int f = 0; f < nf; f++)
    for (int i = off[f]; i < off[f + 1]; i++) {
      const double a = rows[2 * (size_t)i], b = rows[2 * (size_t)i + 1];
      if (!std::isfinite(a) || !std::isfinite(b) || !(b - a > 1e-6)) {
        set_error(std::string(who) + ": scored region " + std::to_string(i - off[f]) + " of file " + std::to_string(f) +
                  " is not finite or not longer than 1e-6 s");
        return DG_EINVAL;
      }
      if (i > off[f] && !(a - rows[2 * (size_t)i - 1] > 1e-6)) {
        set_error(std::string(who) + ": scored region " + std::to_string(i - off[f]) + " of file " + std::to_string(f) +
                  " does not start more than 1e-6 s after the previous one ends");
        return DG_EINVAL;
      }
    }
  if (!r) {
    set_error(std::string(who) + ": null handle");
    return DG_EINVAL;
  }
  r->nf = nf;
  r->rows.assign(rows, rows + 2 * (size_t)S);
  if (nf > 0)
    r->off.assign(off, off + nf + 1);
  else
    r->off.clear();
  return DG_OK;
}

// a scoring call over nf files while regions are set must cover exactly their files (before any launch)
static int regions_check(const char* who, const ScoredRegions& r, int nf) {
  if (r.nf > 0 && r.nf != nf) {
    set_error(std::string(who) + ": scored regions are set for " + std::to_string(r.nf) + " files, the call scores " +
              std::to_string(nf) + " (set them again, or clear them with num_files = 0)");
    return DG_EINVAL;
  }
  return DG_OK;
}

struct dg_sweep {
  int device = 0, M = 0, D = 0, F = 0, K = 0, nw = 1;
  DevBuf hamming, in, centers, active, init, prep, prep_d, maps, header, turns, total;
  DerBufs der;                    // dg_sweep_score
  ScoredRegions regions;          // dg_sweep_set_scored_regions
  int num_sets = 0;               // dg_sweep_set_trial_sets: > 0: emb is [num_sets][N][K][D], trial t reads set trial_set[t]
  std::vector<int32_t> trial_set;
  int seed_nf = 0;                // dg_sweep_set_seeds: > 0: file f's states start from rows [seed_off[f], seed_off[f + 1])
  std::vector<int32_t> seed_off;  // [seed_nf + 1]
  std::vector<double> seeds;      // [seed_off[seed_nf]][D]
  int named_nf = 0;               // dg_sweep_set_identities: > 0: the scoring calls score identification error
  std::vector<int32_t> named;     // [named_nf][32]: per file and reference label, the hypothesis label of the same name or -1
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

extern "C" int dg_sweep_set_scored_regions(dg_sweep* h, int num_files, const double* rows_host,
                                           const int32_t* offsets_host) {
  return set_scored_regions("dg_sweep_set_scored_regions", h ? &h->regions : nullptr, num_files, rows_host, offsets_host);
}

extern "C" int dg_sweep_set_trial_sets(dg_sweep* h, int num_sets, const int32_t* trial_set_host, int T) {
  const char* who = "dg_sweep_set_trial_sets";
  if (num_sets < 0 || num_sets > DG_MAX_OSP_SETS || (num_sets > 0 && (!trial_set_host || T < 1 || T > 65535))) {
    set_error(std::string(who) + ": bad arguments (need 0 <= num_sets <= 64, and 1 <= T <= 65535 trial sets when num_sets > 0)");
    return DG_EINVAL;
  }
  for (int t = 0; num_sets > 0 && t < T; t++)
    if (trial_set_host[t] < 0 || trial_set_host[t] >= num_sets) {
      set_error(std::string(who) + ": trial " + std::to_string(t) + " has set " + std::to_string(trial_set_host[t]) +
                ", outside [0, " + std::to_string(num_sets) + ")");
      return DG_EINVAL;
    }
  if (!h) {
    set_error(std::string(who) + ": null handle");
    return DG_EINVAL;
  }
  h->num_sets = num_sets;
  if (num_sets > 0) h->trial_set.assign(trial_set_host, trial_set_host + T);
  else h->trial_set.clear();
  return DG_OK;
}

extern "C" int dg_sweep_set_seeds(dg_sweep* h, int num_files, const int32_t* offsets_host, const double* centers_host) {
  const char* who = "dg_sweep_set_seeds";
  if (!h) {
    set_error(std::string(who) + ": null handle");
    return DG_EINVAL;
  }
  if (num_files < 0 || (num_files > 0 && !offsets_host)) {
    set_error(std::string(who) + ": bad arguments (need num_files >= 0 and offsets when num_files > 0)");
    return DG_EINVAL;
  }
  if (num_files > 0 && offsets_host[0] != 0) {
    set_error(std::string(who) + ": seed offsets must start at 0");
    return DG_EINVAL;
  }
  for (int f = 0; f < num_files; f++) {
    const int n = offsets_host[f + 1] - offsets_host[f];
    if (n < 0 || n > h->M) {
      set_error(std::string(who) + ": file " + std::to_string(f) + " has " + std::to_string(n) + " centroids (need 0 .. "
                "max_speakers = " + std::to_string(h->M) + "; offsets must not decrease)");
      return DG_EINVAL;
    }
  }
  const int n_total = num_files > 0 ? offsets_host[num_files] : 0;
  if (n_total > 0 && !centers_host) {
    set_error(std::string(who) + ": non-null centroids needed for " + std::to_string(n_total) + " rows");
    return DG_EINVAL;
  }
  const int D = h->D;
  for (int f = 0; f < num_files; f++)   // the rules of dg_multi_open_seeded
    for (int i = offsets_host[f]; i < offsets_host[f + 1]; i++) {
      double ss = 0.0;
      bool finite = true;
      for (int d = 0; d < D; d++) {
        const double x = centers_host[(size_t)i * D + d];
        finite = finite && std::isfinite(x);
        ss += x * x;
      }
      if (!finite || !(ss > 0.0)) {
        set_error(std::string(who) + ": centroid " + std::to_string(i - offsets_host[f]) + " of file " + std::to_string(f) +
                  (finite ? " has a zero norm" : " is not finite"));
        return DG_EINVAL;
      }
    }
  h->seed_nf = num_files;
  if (num_files > 0) h->seed_off.assign(offsets_host, offsets_host + num_files + 1);
  else h->seed_off.clear();
  h->seeds.assign(centers_host, centers_host + (size_t)n_total * D);
  return DG_OK;
}

extern "C" int dg_sweep_set_identities(dg_sweep* h, int num_files, const int32_t* hyp_of_ref_host) {
  const char* who = "dg_sweep_set_identities";
  if (!h) {
    set_error(std::string(who) + ": null handle");
    return DG_EINVAL;
  }
  if (num_files < 0 || (num_files > 0 && !hyp_of_ref_host)) {
    set_error(std::string(who) + ": bad arguments (need num_files >= 0 and a table when num_files > 0)");
    return DG_EINVAL;
  }
  for (int f = 0; f < num_files; f++) {
    unsigned seen = 0;
    for (int r = 0; r < 32; r++) {
      const int g = hyp_of_ref_host[(size_t)f * 32 + r];
      if (g < -1 || g >= h->M) {
        set_error(std::string(who) + ": file " + std::to_string(f) + ", reference label " + std::to_string(r) + ": entry " +
                  std::to_string(g) + " outside [-1, max_speakers = " + std::to_string(h->M) + ")");
        return DG_EINVAL;
      }
      if (g >= 0 && ((seen >> g) & 1u)) {
        set_error(std::string(who) + ": file " + std::to_string(f) + ": hypothesis label " + std::to_string(g) +
                  " is given to two reference labels");
        return DG_EINVAL;
      }
      if (g >= 0) seen |= 1u << g;
    }
  }
  h->named_nf = num_files;
  h->named.assign(hyp_of_ref_host, hyp_of_ref_host + (size_t)num_files * 32);
  return DG_OK;
}

// a scoring call over nf files while identities are set must cover exactly their files (before any launch)
static int identities_check(const char* who, const dg_sweep* h, int nf) {
  if (h->named_nf > 0 && h->named_nf != nf) {
    set_error(std::string(who) + ": identities are set for " + std::to_string(h->named_nf) + " files, the call scores " +
              std::to_string(nf) + " (set them again, or clear them with num_files = 0)");
    return DG_EINVAL;
  }
  return DG_OK;
}

// at most this many (file, trial) states per call: der_hyp runs one warp per (state, label) with up to 32 labels and
// numbers its threads in int32
static const long long DG_SWEEP_MAX_STATES = 1LL << 21;

// chunk offsets [nf + 1] of N chunks: from 0 to N, every file with a chunk
static int check_chunk_offsets(const char* who, int N, int nf, const int32_t* chunk_off) {
  if (chunk_off[0] != 0 || chunk_off[nf] != N) {
    set_error(std::string(who) + ": chunk offsets must start at 0 and end at N");
    return DG_EINVAL;
  }
  for (int f = 0; f < nf; f++)
    if (chunk_off[f + 1] <= chunk_off[f]) {
      set_error(std::string(who) + ": file " + std::to_string(f) + " has no chunks (offsets must increase)");
      return DG_EINVAL;
    }
  return DG_OK;
}

// the argument checks dg_sweep_run(_files) and dg_sweep_score(_files) share (before any launch); chunk_off [nf + 1] splits
// the N chunks into the files' ranges
static int sweep_check(const char* who, dg_sweep* h, const float* seg_dev, const float* emb_dev, int N, int nf,
                       const int32_t* chunk_off, const double* params_host, int T, const int32_t* plan_host) {
  if (!h || !seg_dev || !emb_dev || !params_host || !plan_host || N < 1 || T < 1 || T > 65535 || nf < 1 || !chunk_off) {
    set_error(std::string(who) + ": bad arguments (need N >= 1, 1 <= T <= 65535, num_files >= 1, non-null buffers)");
    return DG_EINVAL;
  }
  if ((long long)nf * T > DG_SWEEP_MAX_STATES) {
    set_error(std::string(who) + ": " + std::to_string((long long)nf * T) + " (file, trial) states; at most " +
              std::to_string(DG_SWEEP_MAX_STATES) + " per call");
    return DG_EINVAL;
  }
  if (h->num_sets > 0 && (int)h->trial_set.size() != T) {
    set_error(std::string(who) + ": trial sets are set for " + std::to_string(h->trial_set.size()) + " trials, the call runs " +
              std::to_string(T) + " (set them again, or clear them with num_sets = 0)");
    return DG_EINVAL;
  }
  if (h->seed_nf > 0 && h->seed_nf != nf) {
    set_error(std::string(who) + ": seeds are set for " + std::to_string(h->seed_nf) + " files, the call clusters " +
              std::to_string(nf) + " (set them again, or clear them with num_files = 0)");
    return DG_EINVAL;
  }
  int rc;
  if ((rc = check_chunk_offsets(who, N, nf, chunk_off))) return rc;
  for (int i = 0; i < 3 * T; i++)
    if (!std::isfinite(params_host[i])) {
      set_error(std::string(who) + ": trial " + std::to_string(i / 3) + " has a parameter that is not finite");
      return DG_EINVAL;
    }
  return DG_OK;
}

// The launch order of the nf * T (file, trial) states, states [nf * T][2] = {file, trial}: longest file first (equal lengths
// in file order), then trial.  A state's time is its file's chunk count; when the states outnumber the resident CTAs, the
// long ones start in the first wave and the last wave holds short ones.
static void sweep_state_order(int nf, const int32_t* chunk_off, int T, int32_t* states) {
  std::vector<int> order(nf);
  for (int f = 0; f < nf; f++) order[f] = f;
  std::stable_sort(order.begin(), order.end(),
                   [&](int a, int b) { return chunk_off[a + 1] - chunk_off[a] > chunk_off[b + 1] - chunk_off[b]; });
  size_t i = 0;
  for (int f : order)
    for (int t = 0; t < T; t++, i++) {
      states[2 * i] = f;
      states[2 * i + 1] = t;
    }
}

extern "C" int dg_sweep_state_order(int num_files, const int32_t* chunk_offsets_host, int T, int32_t* states_host) {
  if (num_files < 1 || T < 1 || !chunk_offsets_host || !states_host) {
    set_error("dg_sweep_state_order: bad arguments (need num_files >= 1, T >= 1, non-null buffers)");
    return DG_EINVAL;
  }
  sweep_state_order(num_files, chunk_offsets_host, T, states_host);
  return DG_OK;
}

// pinned output layout of sweep_cluster_post over S states: error flags [S][2], then header [T][N][4], turn count, turn prefix
static TurnOut sweep_out(int S, int T, int N) { return {(size_t)S * 8, (size_t)T * N * 16}; }

// Clustering + post-path of T trials over the nf files whose chunks [chunk_off[f], chunk_off[f + 1]) make up the N chunks:
// header [T][N][4] and turns stay on the device (h->header, h->turns), the turn count comes back in *total.  with_header: the
// header and a prefix of the turns travel to the pinned buffer in the same copy as the count (sweep_out layout).  The plan
// is the files' plans, each that of a fresh stream, concatenated: a chunk's aggregated buffers are the nw - 1 chunks before
// it at most, never those of the previous file (check_file_plans: chunk c reads chunks c - (nb - 1) .. c, nb <= its index in
// its file + 1), so the post-path runs over all N chunks at once.  Synchronises `st`.
//
// With vchunk_host (the sweep over several latencies): the nf "files" are units, the clustering runs over them as above, and
// the post-path runs over Nv virtual chunks instead, virtual chunk c being real chunk vchunk_host[c]; the plan [Nv][stride] and
// the header [T][Nv][4] are over the virtual chunks.  Without it Nv = N, virtual chunk c being chunk c.  used [nf] (or null:
// all): the units whose (unit, trial) states are clustered; the maps of the others' chunks are left unwritten.
static int sweep_cluster_post(dg_sweep* h, const float* seg_dev, const float* emb_dev, int N, int nf, const int32_t* chunk_off,
                              const double* params_host, int T, const int32_t* plan_host, int32_t* maps_dev,
                              double* centers_dev, bool with_header, cudaStream_t st, unsigned int* total_out,
                              int Nv = 0, const int32_t* vchunk_host = nullptr, const std::vector<char>* used = nullptr) {
  if (!vchunk_host) Nv = N;
  // the launch order of the (file, trial) states, without those of units nobody reads
  std::vector<int32_t> states((size_t)nf * T * 2);
  sweep_state_order(nf, chunk_off, T, states.data());
  if (used) {
    size_t k = 0;
    for (size_t i = 0; i < (size_t)nf * T; i++)
      if ((*used)[states[2 * i]]) {
        states[2 * k] = states[2 * i];
        states[2 * k + 1] = states[2 * i + 1];
        k++;
      }
    states.resize(2 * k);
  }
  // state s = f T + t owns centroid table, active flags and error pair s (cluster.cu), so those are sized for all nf T states
  // whichever of them run; the launch runs S_run
  const int stride = 4 + h->nw, M = h->M, D = h->D, K = h->K, F = h->F, S = nf * T, S_run = (int)(states.size() / 2);
  // with trial sets (dg_sweep_set_trial_sets) a trial row is {tau, rho, delta, set}, and the prep rows are per set
  const int G = h->num_sets, PS = G > 0 ? 4 : 3;
  // host -> device, one copy: params [T][PS], taus [T], states [S_run][2] (launch order), plan [Nv][stride], chunk offsets
  // [nf + 1], then with vchunk_host the virtual chunk table [Nv], then with seeds (dg_sweep_set_seeds) their offsets [nf + 1]
  // and, at the next multiple of 8 bytes, their centroids [n][D]
  const size_t params_b = (size_t)T * PS * 8, taus_b = (size_t)T * 8, states_b = (size_t)S_run * 8, plan_b = (size_t)Nv * stride * 4;
  const size_t off_b = (size_t)(nf + 1) * 4, vchunk_b = vchunk_host ? (size_t)Nv * 4 : 0;
  const bool seeded = h->seed_nf > 0;
  const size_t base_b = params_b + taus_b + states_b + plan_b + off_b + vchunk_b;
  const size_t soff_b = seeded ? off_b : 0, seeds_at = (base_b + soff_b + 7) & ~(size_t)7;
  const size_t in_b = seeded ? seeds_at + h->seeds.size() * 8 : base_b;
  const TurnOut lay = sweep_out(S, T, Nv);
  const size_t init_b = lay.at, header_b = lay.header_bytes;
  // the device turn buffer starts at a guess and grows to the true count (the kernel counts every turn, writes those that fit)
  const size_t turn_guess = std::max<size_t>((size_t)T * Nv * 8, (size_t)DG_POST_PREFIX);
  if (h->in.ensure(in_b) || h->centers.ensure((size_t)S * M * D * 8) || h->active.ensure((size_t)S * 32 * 4) ||
      h->init.ensure(init_b) || h->prep.ensure(cluster_prep_floats(N, K) * 4 * std::max(G, 1) + 16) ||
      h->prep_d.ensure(cluster_prep_doubles(N, K) * 8 * std::max(G, 1) + 16) || (!maps_dev && h->maps.ensure((size_t)T * N * K * 4)) ||
      h->header.ensure(header_b) || h->turns.ensure(turn_guess * 4) || h->pin.ensure(std::max(in_b, lay.end())))
    return DG_ECUDA;
  unsigned char* pin = h->pin.as<unsigned char>();
  double* p_taus = reinterpret_cast<double*>(pin + params_b);
  if (G > 0) {
    double* rows = reinterpret_cast<double*>(pin);
    for (int t = 0; t < T; t++) {
      for (int j = 0; j < 3; j++) rows[4 * t + j] = params_host[3 * t + j];
      rows[4 * t + 3] = (double)h->trial_set[t];
    }
  } else {
    memcpy(pin, params_host, params_b);
  }
  for (int t = 0; t < T; t++) p_taus[t] = params_host[3 * t];
  memcpy(pin + params_b + taus_b, states.data(), states_b);
  memcpy(pin + params_b + taus_b + states_b, plan_host, plan_b);
  memcpy(pin + params_b + taus_b + states_b + plan_b, chunk_off, off_b);
  if (vchunk_host) memcpy(pin + params_b + taus_b + states_b + plan_b + off_b, vchunk_host, vchunk_b);
  if (seeded) {
    memcpy(pin + base_b, h->seed_off.data(), soff_b);
    if (!h->seeds.empty()) memcpy(pin + seeds_at, h->seeds.data(), h->seeds.size() * 8);
  }
  unsigned char* din = h->in.as<unsigned char>();
  DG_CUDA(cudaMemcpyAsync(din, pin, in_b, cudaMemcpyHostToDevice, st));
  const double* d_params = reinterpret_cast<const double*>(din);
  const double* d_taus = reinterpret_cast<const double*>(din + params_b);
  const int2* d_states = reinterpret_cast<const int2*>(din + params_b + taus_b);
  const int32_t* d_plan = reinterpret_cast<const int32_t*>(din + params_b + taus_b + states_b);
  const int* d_off = reinterpret_cast<const int*>(din + params_b + taus_b + states_b + plan_b);
  int32_t* maps = maps_dev ? maps_dev : h->maps.as<int32_t>();
  // every state starts empty (reference: a new OnlineSpeakerClustering per trial and file)
  DG_CUDA(cudaMemsetAsync(h->centers.p, 0, (size_t)S * M * D * 8, st));
  DG_CUDA(cudaMemsetAsync(h->active.p, 0, (size_t)S * 32 * 4, st));
  DG_CUDA(cudaMemsetAsync(h->init.p, 0, init_b, st));
  int rc;
  // a seeded file's states start from its known centroids instead (dg_multi_open_seeded's state)
  if (seeded && (rc = launch_sweep_seed(reinterpret_cast<const int*>(din + base_b), reinterpret_cast<const double*>(din + seeds_at),
                                        nf, T, M, D, h->centers.as<double>(), h->active.as<int>(), h->init.as<int>(), st)))
    return rc;
  ClusterParams p{};
  p.M = M;
  p.D = D;
  p.metric = 0;
  if (G > 0)
    rc = launch_cluster_sweep_sets(p, d_params, T, d_states, S_run, d_off, seg_dev, emb_dev, G, N, F, K, h->centers.as<double>(),
                                   h->active.as<int>(), h->init.as<int>(), h->prep.as<float>(), h->prep_d.as<double>(), maps, st);
  else
    rc = launch_cluster_sweep(p, d_params, T, d_states, S_run, d_off, seg_dev, emb_dev, N, F, K, h->centers.as<double>(),
                              h->active.as<int>(), h->init.as<int>(), h->prep.as<float>(), h->prep_d.as<double>(), maps, st);
  if (rc) return rc;
  if (centers_dev)
    DG_CUDA(cudaMemcpyAsync(centers_dev, h->centers.p, (size_t)S * M * D * 8, cudaMemcpyDeviceToDevice, st));
  unsigned int total = 0;
  for (int attempt = 0; attempt < 2; attempt++) {
    const int cap = (int)std::min<size_t>(h->turns.bytes / 4, (size_t)INT32_MAX);
    DG_CUDA(cudaMemsetAsync(h->total.p, 0, 4, st));
    if ((rc = launch_post_virtual(seg_dev, maps, N, vchunk_host ? reinterpret_cast<const int32_t*>(d_off + nf + 1) : nullptr, Nv,
                                  F, K, M, h->nw, d_plan, stride, h->hamming.as<double>(), d_taus, T, h->header.as<int32_t>(),
                                  h->turns.as<uint32_t>(), cap, h->total.as<unsigned int>(), st)))
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
  for (int s = 0; s < S; s++)
    if (flags[2 * s + 1]) {
      set_error("Cannot update unknown centers");   // reference clustering.py:98 (AssertionError)
      return DG_EINVAL;
    }
  *total_out = total;
  return DG_OK;
}

static int sweep_run(const char* who, dg_sweep* h, const float* seg_dev, const float* emb_dev, int N, int nf,
                     const int32_t* chunk_off, const double* params_host, int T, const int32_t* plan_host, int32_t* maps_dev,
                     double* centers_dev, int32_t* header_host, uint32_t* turns_host, int turn_cap_host, int* n_turns,
                     void* stream) {
  if (!header_host || !turns_host) {
    set_error(std::string(who) + ": bad arguments (need N >= 1, 1 <= T <= 65535, non-null buffers)");
    return DG_EINVAL;
  }
  int rc;
  if ((rc = sweep_check(who, h, seg_dev, emb_dev, N, nf, chunk_off, params_host, T, plan_host)) ||
      (rc = check_file_plans(who, plan_host, nf, chunk_off, h->nw, h->F)))
    return rc;
  DG_CUDA(cudaSetDevice(h->device));
  cudaStream_t st = (cudaStream_t)stream;
  unsigned int total = 0;
  if ((rc = sweep_cluster_post(h, seg_dev, emb_dev, N, nf, chunk_off, params_host, T, plan_host, maps_dev, centers_dev, true,
                               st, &total)))
    return rc;
  return download_turns(who, h->pin.as<unsigned char>(), sweep_out(nf * T, T, N), h->turns.as<uint32_t>(), header_host,
                        turns_host, turn_cap_host, n_turns, st);
}

extern "C" int dg_sweep_run(dg_sweep* h, const float* seg_dev, const float* emb_dev, int N, const double* params_host, int T,
                            const int32_t* plan_host, int32_t* maps_dev, double* centers_dev, int32_t* header_host,
                            uint32_t* turns_host, int turn_cap_host, int* n_turns, void* stream) {
  const int32_t off[2] = {0, N};
  return sweep_run("dg_sweep_run", h, seg_dev, emb_dev, N, 1, off, params_host, T, plan_host, maps_dev, centers_dev,
                   header_host, turns_host, turn_cap_host, n_turns, stream);
}

extern "C" int dg_sweep_run_files(dg_sweep* h, const float* seg_dev, const float* emb_dev, int N, int num_files,
                                  const int32_t* chunk_offsets_host, const double* params_host, int T,
                                  const int32_t* plan_host, int32_t* maps_dev, double* centers_dev, int32_t* header_host,
                                  uint32_t* turns_host, int turn_cap_host, int* n_turns, void* stream) {
  return sweep_run("dg_sweep_run_files", h, seg_dev, emb_dev, N, num_files, chunk_offsets_host, params_host, T, plan_host,
                   maps_dev, centers_dev, header_host, turns_host, turn_cap_host, n_turns, stream);
}

// the reference rows of one file: finite, start < end, labels in [0, R), each label's rows in time order without overlap
static int sweep_check_reference(const char* who, const double* ref_host, const int32_t* ref_label_host, int S, int R) {
  if (R < 0 || R > 32 || S < 0 || (S > 0 && (!ref_host || !ref_label_host))) {
    set_error(std::string(who) + ": need 0 <= reference labels <= 32, rows >= 0, non-null reference arrays");
    return DG_EINVAL;
  }
  double last[32];
  for (int r = 0; r < 32; r++) last[r] = -INFINITY;
  for (int i = 0; i < S; i++) {
    const double a = ref_host[2 * i], b = ref_host[2 * i + 1];
    const int r = ref_label_host[i];
    if (r < 0 || r >= R) {
      set_error(std::string(who) + ": reference row " + std::to_string(i) + " has a label outside [0, R)");
      return DG_EINVAL;
    }
    if (!std::isfinite(a) || !std::isfinite(b) || !(a < b)) {
      set_error(std::string(who) + ": reference row " + std::to_string(i) + " is not finite, empty or reversed");
      return DG_EINVAL;
    }
    if (a < last[r]) {
      set_error(std::string(who) + ": reference row " + std::to_string(i) +
                " is out of order or overlaps an earlier row of its label");
      return DG_EINVAL;
    }
    last[r] = b;
  }
  return DG_OK;
}

// The der_hyp -> der_scan -> der_score sequence over a post-path result already on the device (header [T][N][4] and `total`
// turns, M labels): the DER components comp [nf][T][5] of every (file, trial) against the file's reference rows
// [ref_off[f], ref_off[f + 1]) with R[f] labels, the arguments checked by the caller.  With regions (nf files), der_score
// crops each hypothesis to its file's scored pieces; the reference rows come cropped.  Uses the pinned buffer `pinbuf`;
// synchronises `st`.
static int der_components(const char* who, DerBufs& b, PinnedBuf& pinbuf, const int32_t* header_dev, const uint32_t* turns_dev,
                          unsigned int total, int N, int nf, const int32_t* chunk_off, int T, int M,
                          const double* out_start_host, const double* out_res_host, const double* shift_host, double collar,
                          const double* ref_host, const int32_t* ref_label_host, const int32_t* ref_off, const int32_t* R_host,
                          double* components_host, int32_t* hyp_offsets_dev, double* hyp_segments_dev, int hyp_cap,
                          cudaStream_t st, const ScoredRegions* regions = nullptr, const int32_t* named = nullptr) {
  int rc;
  const int NTM = nf * T * M, S = ref_off[nf];
  const bool crop = regions && regions->nf > 0;
  // host -> device, one copy: out_start [N], out_res [N], shifts [nf], reference segments [S][2] grouped by label within each
  // file, label offsets [nf][DER_ROFF], label counts [nf], chunk offsets [nf + 1], then with regions the scored pieces [U][2]
  // (at the next multiple of 8 bytes) and their offsets [nf + 1], then with named (identification error) its table [nf][32]
  const size_t times_b = (size_t)N * 16, shift_b = (size_t)nf * 8, rseg_b = (size_t)S * 16;
  const size_t roff_b = (size_t)nf * DER_ROFF * 4, R_b = (size_t)nf * 4, off_b = (size_t)(nf + 1) * 4;
  const size_t base_b = times_b + shift_b + rseg_b + roff_b + R_b + off_b, useg_at = (base_b + 7) & ~(size_t)7;
  const size_t useg_b = crop ? regions->rows.size() * 8 : 0, uoff_b = crop ? (size_t)(nf + 1) * 4 : 0;
  const size_t named_at = crop ? useg_at + useg_b + uoff_b : base_b, named_b = named ? (size_t)nf * 32 * 4 : 0;
  const size_t in_b = named_at + named_b, comp_b = (size_t)nf * T * 40;
  if (b.in.ensure(in_b) || b.hoff.ensure((size_t)(NTM + 1) * 4) || b.hseg.ensure((size_t)std::max(total, 1u) * 16) ||
      b.comp.ensure(comp_b) || pinbuf.ensure(std::max(in_b, comp_b + 16)))
    return DG_ECUDA;
  unsigned char* pin = pinbuf.as<unsigned char>();
  memcpy(pin, out_start_host, (size_t)N * 8);
  memcpy(pin + (size_t)N * 8, out_res_host, (size_t)N * 8);
  memcpy(pin + times_b, shift_host, shift_b);
  double* rseg = reinterpret_cast<double*>(pin + times_b + shift_b);
  int32_t* roff_all = reinterpret_cast<int32_t*>(pin + times_b + shift_b + rseg_b);
  memcpy(pin + times_b + shift_b + rseg_b + roff_b, R_host, R_b);
  memcpy(pin + times_b + shift_b + rseg_b + roff_b + R_b, chunk_off, off_b);
  if (crop) {
    if (useg_b) memcpy(pin + useg_at, regions->rows.data(), useg_b);
    memcpy(pin + useg_at + useg_b, regions->off.data(), uoff_b);
  }
  if (named) memcpy(pin + named_at, named, named_b);
  for (int f = 0; f < nf; f++) {
    const int a = ref_off[f], n = ref_off[f + 1] - a, R = R_host[f];
    int32_t* roff = roff_all + (size_t)f * DER_ROFF;
    for (int r = 0; r < DER_ROFF; r++) roff[r] = 0;
    for (int i = 0; i < n; i++) roff[ref_label_host[a + i] + 1]++;
    roff[0] = a;
    for (int r = 0; r < R; r++) roff[r + 1] += roff[r];
    int fill[32];
    for (int r = 0; r < R; r++) fill[r] = roff[r];
    for (int i = 0; i < n; i++) {     // stable: each label keeps its rows' order
      const int o = fill[ref_label_host[a + i]]++;
      rseg[2 * (size_t)o] = ref_host[2 * (size_t)(a + i)];
      rseg[2 * (size_t)o + 1] = ref_host[2 * (size_t)(a + i) + 1];
    }
  }
  unsigned char* din = b.in.as<unsigned char>();
  DG_CUDA(cudaMemcpyAsync(din, pin, in_b, cudaMemcpyHostToDevice, st));
  const double* d_start = reinterpret_cast<const double*>(din);
  const double* d_res = d_start + N;
  const double* d_shift = reinterpret_cast<const double*>(din + times_b);
  const double* d_rseg = reinterpret_cast<const double*>(din + times_b + shift_b);
  const int* d_roff = reinterpret_cast<const int*>(din + times_b + shift_b + rseg_b);
  const int* d_R = reinterpret_cast<const int*>(din + times_b + shift_b + rseg_b + roff_b);
  const int* d_off = reinterpret_cast<const int*>(din + times_b + shift_b + rseg_b + roff_b + R_b);
  const double* d_useg = crop ? reinterpret_cast<const double*>(din + useg_at) : nullptr;
  const int* d_uoff = crop ? reinterpret_cast<const int*>(din + useg_at + useg_b) : nullptr;
  const int* d_named = named ? reinterpret_cast<const int*>(din + named_at) : nullptr;
  int* hoff = b.hoff.as<int>();
  if ((rc = launch_der_hyp_count(header_dev, turns_dev, nf, d_off, T, N, M, d_start, d_res, d_shift, collar, hoff, st)) ||
      (rc = launch_der_hyp_write(header_dev, turns_dev, nf, d_off, T, N, M, d_start, d_res, d_shift, collar, hoff,
                                 b.hseg.as<double>(), hyp_segments_dev, hyp_cap, st)) ||
      (rc = launch_der_score(hoff, b.hseg.as<double>(), nf, T, M, d_roff, d_R, d_rseg, b.comp.as<double>(), st, d_uoff,
                             d_useg, d_named)))
    return rc;
  if (hyp_offsets_dev) DG_CUDA(cudaMemcpyAsync(hyp_offsets_dev, hoff, (size_t)(NTM + 1) * 4, cudaMemcpyDeviceToDevice, st));
  DG_CUDA(cudaMemcpyAsync(pin, b.comp.p, comp_b, cudaMemcpyDeviceToHost, st));
  DG_CUDA(cudaMemcpyAsync(pin + comp_b, hoff + NTM, 4, cudaMemcpyDeviceToHost, st));
  DG_CUDA(cudaStreamSynchronize(st));
  memcpy(components_host, pin, comp_b);
  int n_seg = 0;
  memcpy(&n_seg, pin + comp_b, 4);
  if (hyp_segments_dev && n_seg > hyp_cap) {
    set_error(std::string(who) + ": hypothesis segment buffer too small (" + std::to_string(n_seg) + " segments)");
    return DG_EINVAL;
  }
  return DG_OK;
}

// the scoring arguments of dg_sweep_score(_files) and dg_sweep_score_latencies over N chunks in nf files (before any launch)
static int score_check(const char* who, int N, int nf, const double* out_start_host, const double* out_res_host,
                       const double* shift_host, double collar, const double* ref_host, const int32_t* ref_label_host,
                       const int32_t* ref_off, const int32_t* R_host, const double* components_host, int hyp_cap) {
  int rc;
  if (!out_start_host || !out_res_host || !components_host || hyp_cap < 0 || !shift_host || !std::isfinite(collar) ||
      collar < 0) {
    set_error(std::string(who) + ": bad arguments (need chunk times, a components buffer, finite shift, finite collar >= 0, "
              "hyp_cap >= 0)");
    return DG_EINVAL;
  }
  for (int f = 0; f < nf; f++)
    if (!std::isfinite(shift_host[f])) {
      set_error(std::string(who) + ": the shift of file " + std::to_string(f) + " is not finite");
      return DG_EINVAL;
    }
  for (int c = 0; c < N; c++)
    if (!std::isfinite(out_start_host[c]) || !std::isfinite(out_res_host[c])) {
      set_error(std::string(who) + ": chunk " + std::to_string(c) + " has an output time that is not finite");
      return DG_EINVAL;
    }
  if (!ref_off || !R_host || ref_off[0] != 0) {
    set_error(std::string(who) + ": need reference row offsets starting at 0 and label counts");
    return DG_EINVAL;
  }
  for (int f = 0; f < nf; f++)
    if (ref_off[f + 1] < ref_off[f]) {
      set_error(std::string(who) + ": rows >= 0 (reference row offsets of file " + std::to_string(f) + " decrease)");
      return DG_EINVAL;
    }
  const int S = ref_off[nf];
  if (S > 0 && (!ref_host || !ref_label_host)) {
    set_error(std::string(who) + ": non-null reference arrays needed for " + std::to_string(S) + " rows");
    return DG_EINVAL;
  }
  for (int f = 0; f < nf; f++)
    if ((rc = sweep_check_reference(who, S > 0 ? ref_host + 2 * (size_t)ref_off[f] : nullptr,
                                    S > 0 ? ref_label_host + ref_off[f] : nullptr, ref_off[f + 1] - ref_off[f], R_host[f])))
      return rc;
  return DG_OK;
}

// dg_sweep_score(_files): the clustering and post-path of sweep_cluster_post, then the DER components of every (file, trial)
// against the file's reference rows [ref_off[f], ref_off[f + 1]) with R[f] labels
static int sweep_score(const char* who, dg_sweep* h, const float* seg_dev, const float* emb_dev, int N, int nf,
                       const int32_t* chunk_off, const double* params_host, int T, const int32_t* plan_host,
                       const double* out_start_host, const double* out_res_host, const double* shift_host, double collar,
                       const double* ref_host, const int32_t* ref_label_host, const int32_t* ref_off, const int32_t* R_host,
                       double* components_host, int32_t* hyp_offsets_dev, double* hyp_segments_dev, int hyp_cap,
                       void* stream) {
  int rc;
  if ((rc = sweep_check(who, h, seg_dev, emb_dev, N, nf, chunk_off, params_host, T, plan_host)) ||
      (rc = check_file_plans(who, plan_host, nf, chunk_off, h->nw, h->F)) ||
      (rc = score_check(who, N, nf, out_start_host, out_res_host, shift_host, collar, ref_host, ref_label_host, ref_off,
                        R_host, components_host, hyp_cap)) ||
      (rc = regions_check(who, h->regions, nf)) || (rc = identities_check(who, h, nf)))
    return rc;
  DG_CUDA(cudaSetDevice(h->device));
  cudaStream_t st = (cudaStream_t)stream;
  unsigned int total = 0;
  if ((rc = sweep_cluster_post(h, seg_dev, emb_dev, N, nf, chunk_off, params_host, T, plan_host, nullptr, nullptr, false, st,
                               &total)))
    return rc;
  return der_components(who, h->der, h->pin, h->header.as<int32_t>(), h->turns.as<uint32_t>(), total, N, nf, chunk_off, T,
                        h->M, out_start_host, out_res_host, shift_host, collar, ref_host, ref_label_host, ref_off, R_host,
                        components_host, hyp_offsets_dev, hyp_segments_dev, hyp_cap, st, &h->regions,
                        h->named_nf > 0 ? h->named.data() : nullptr);
}

extern "C" int dg_sweep_score(dg_sweep* h, const float* seg_dev, const float* emb_dev, int N, const double* params_host,
                              int T, const int32_t* plan_host, const double* out_start_host, const double* out_res_host,
                              double shift, double collar, const double* ref_host, const int32_t* ref_label_host, int S,
                              int R, double* components_host, int32_t* hyp_offsets_dev, double* hyp_segments_dev,
                              int hyp_cap, void* stream) {
  const int32_t off[2] = {0, N}, ref_off[2] = {0, S};
  return sweep_score("dg_sweep_score", h, seg_dev, emb_dev, N, 1, off, params_host, T, plan_host, out_start_host,
                     out_res_host, &shift, collar, ref_host, ref_label_host, ref_off, &R, components_host, hyp_offsets_dev,
                     hyp_segments_dev, hyp_cap, stream);
}

extern "C" int dg_sweep_score_files(dg_sweep* h, const float* seg_dev, const float* emb_dev, int N, int num_files,
                                    const int32_t* chunk_offsets_host, const double* params_host, int T,
                                    const int32_t* plan_host, const double* out_start_host, const double* out_res_host,
                                    const double* shifts_host, double collar, const double* ref_host,
                                    const int32_t* ref_label_host, const int32_t* ref_offsets_host,
                                    const int32_t* ref_label_counts_host, double* components_host, int32_t* hyp_offsets_dev,
                                    double* hyp_segments_dev, int hyp_cap, void* stream) {
  return sweep_score("dg_sweep_score_files", h, seg_dev, emb_dev, N, num_files, chunk_offsets_host, params_host, T, plan_host,
                     out_start_host, out_res_host, shifts_host, collar, ref_host, ref_label_host, ref_offsets_host,
                     ref_label_counts_host, components_host, hyp_offsets_dev, hyp_segments_dev, hyp_cap, stream);
}

// ============================================================================= sweeps over several latencies
// A file's windows at a smaller latency are a prefix of its windows at a larger one (same left padding), so the network
// outputs of a *unit* -- the windows of a file at the largest latency of a group whose outputs are its prefixes bit for bit
// (the host groups them, tune.LatencyUnits) -- serve every latency of the group.  A *virtual file* is one (latency, file)
// pair: the first chunks of its unit.  Its *virtual chunks* carry the plan row, output times and timestamp shift of that
// latency; the clustering runs over the units (it is causal and never reads the latency), the post-path and the scoring over
// the virtual chunks.

// The virtual layout over N real chunks in nu units (unit_off [nu + 1]): virtual file v holds virtual chunks [voff[v],
// voff[v + 1]) of Nv, which must be the real chunks u0, u0 + 1, ... of one unit starting at its first chunk u0, inside it; the
// plan row [4 + nw] of its i-th virtual chunk is that of the i-th chunk of a fresh stream (check_plan_row).  used (or null)
// receives [nu]: whether a virtual file starts at unit u.  Host only.
static int check_virtual(const char* who, int N, int nu, const int32_t* unit_off, int Nv, int nvf, const int32_t* vchunk,
                         const int32_t* voff, const int32_t* plan, int nw, int F, std::vector<char>* used = nullptr) {
  if (N < 1 || nu < 1 || Nv < 1 || nvf < 1 || nw < 1 || F < 1 || !unit_off || !vchunk || !voff || !plan) {
    set_error(std::string(who) + ": bad virtual layout arguments (need chunks, units, virtual chunks and files >= 1, "
              "non-null tables)");
    return DG_EINVAL;
  }
  int rc;
  if ((rc = check_chunk_offsets(who, N, nu, unit_off)) || (rc = check_chunk_offsets(who, Nv, nvf, voff))) return rc;
  const int stride = 4 + nw;
  if (used) used->assign(nu, 0);
  for (int v = 0; v < nvf; v++) {
    const int a = voff[v], n = voff[v + 1] - a, c0 = vchunk[a];
    const int u = (int)(std::upper_bound(unit_off, unit_off + nu + 1, c0) - unit_off) - 1;
    if (c0 < 0 || c0 >= N || u < 0 || u >= nu || unit_off[u] != c0) {
      set_error(std::string(who) + ": virtual file " + std::to_string(v) + " does not start at the first chunk of a unit");
      return DG_EINVAL;
    }
    if (n > unit_off[u + 1] - c0) {
      set_error(std::string(who) + ": virtual file " + std::to_string(v) + " crosses into the next unit");
      return DG_EINVAL;
    }
    if (used) (*used)[u] = 1;
    for (int i = 0; i < n; i++) {
      if (vchunk[a + i] != c0 + i) {
        set_error(std::string(who) + ": virtual file " + std::to_string(v) + " is not a run of consecutive chunks of its unit");
        return DG_EINVAL;
      }
      if ((rc = check_plan_row(who, plan + (size_t)(a + i) * stride, a + i, nw, i, F))) return rc;
    }
  }
  return DG_OK;
}

extern "C" int dg_sweep_check_latencies(int N, int num_units, const int32_t* unit_offsets_host, int num_virtual,
                                        int num_virtual_files, const int32_t* vchunk_host,
                                        const int32_t* virtual_offsets_host, const int32_t* plan_host, int num_windows,
                                        int frames) {
  return check_virtual("dg_sweep_check_latencies", N, num_units, unit_offsets_host, num_virtual, num_virtual_files,
                       vchunk_host, virtual_offsets_host, plan_host, num_windows, frames);
}

// the checks dg_sweep_run_latencies and dg_sweep_score_latencies share: sweep_check over the units, the virtual layout, and
// at most DG_SWEEP_MAX_STATES (virtual file, trial) states for the scoring; used [nu]: the units the virtual files read
static int latency_check(const char* who, dg_sweep* h, const float* seg_dev, const float* emb_dev, int N, int nu,
                         const int32_t* unit_off, int Nv, int nvf, const int32_t* vchunk, const int32_t* voff,
                         const double* params_host, int T, const int32_t* plan_host, std::vector<char>& used) {
  int rc;
  if ((rc = sweep_check(who, h, seg_dev, emb_dev, N, nu, unit_off, params_host, T, plan_host))) return rc;
  if ((long long)nvf * T > DG_SWEEP_MAX_STATES) {
    set_error(std::string(who) + ": " + std::to_string((long long)nvf * T) + " (virtual file, trial) states; at most " +
              std::to_string(DG_SWEEP_MAX_STATES) + " per call");
    return DG_EINVAL;
  }
  return check_virtual(who, N, nu, unit_off, Nv, nvf, vchunk, voff, plan_host, h->nw, h->F, &used);
}

extern "C" int dg_sweep_run_latencies(dg_sweep* h, const float* seg_dev, const float* emb_dev, int N, int num_units,
                                      const int32_t* unit_offsets_host, int num_virtual, int num_virtual_files,
                                      const int32_t* vchunk_host, const int32_t* virtual_offsets_host,
                                      const double* params_host, int T, const int32_t* plan_host, int32_t* maps_dev,
                                      int32_t* header_host, uint32_t* turns_host, int turn_cap_host, int* n_turns,
                                      void* stream) {
  const char* who = "dg_sweep_run_latencies";
  std::vector<char> used;
  int rc;
  if ((rc = latency_check(who, h, seg_dev, emb_dev, N, num_units, unit_offsets_host, num_virtual, num_virtual_files,
                          vchunk_host, virtual_offsets_host, params_host, T, plan_host, used)))
    return rc;
  if (!header_host || !turns_host) {
    set_error(std::string(who) + ": bad arguments (need non-null header and turn buffers)");
    return DG_EINVAL;
  }
  DG_CUDA(cudaSetDevice(h->device));
  cudaStream_t st = (cudaStream_t)stream;
  unsigned int total = 0;
  if ((rc = sweep_cluster_post(h, seg_dev, emb_dev, N, num_units, unit_offsets_host, params_host, T, plan_host, maps_dev,
                               nullptr, true, st, &total, num_virtual, vchunk_host, &used)))
    return rc;
  return download_turns(who, h->pin.as<unsigned char>(), sweep_out(num_units * T, T, num_virtual), h->turns.as<uint32_t>(),
                        header_host, turns_host, turn_cap_host, n_turns, st);
}

extern "C" int dg_sweep_score_latencies(dg_sweep* h, const float* seg_dev, const float* emb_dev, int N, int num_units,
                                        const int32_t* unit_offsets_host, int num_virtual, int num_virtual_files,
                                        const int32_t* vchunk_host, const int32_t* virtual_offsets_host,
                                        const double* params_host, int T, const int32_t* plan_host,
                                        const double* out_start_host, const double* out_res_host, const double* shifts_host,
                                        double collar, const double* ref_host, const int32_t* ref_label_host,
                                        const int32_t* ref_offsets_host, const int32_t* ref_label_counts_host,
                                        double* components_host, void* stream) {
  const char* who = "dg_sweep_score_latencies";
  std::vector<char> used;
  int rc;
  if ((rc = latency_check(who, h, seg_dev, emb_dev, N, num_units, unit_offsets_host, num_virtual, num_virtual_files,
                          vchunk_host, virtual_offsets_host, params_host, T, plan_host, used)))
    return rc;
  const int Nv = num_virtual, nvf = num_virtual_files;
  if ((rc = score_check(who, Nv, nvf, out_start_host, out_res_host, shifts_host, collar, ref_host, ref_label_host,
                        ref_offsets_host, ref_label_counts_host, components_host, 0)) ||
      (rc = regions_check(who, h->regions, nvf)) || (rc = identities_check(who, h, nvf)))
    return rc;
  DG_CUDA(cudaSetDevice(h->device));
  cudaStream_t st = (cudaStream_t)stream;
  unsigned int total = 0;
  if ((rc = sweep_cluster_post(h, seg_dev, emb_dev, N, num_units, unit_offsets_host, params_host, T, plan_host, nullptr,
                               nullptr, false, st, &total, Nv, vchunk_host, &used)))
    return rc;
  return der_components(who, h->der, h->pin, h->header.as<int32_t>(), h->turns.as<uint32_t>(), total, Nv, nvf,
                        virtual_offsets_host, T, h->M, out_start_host, out_res_host, shifts_host, collar, ref_host,
                        ref_label_host, ref_offsets_host, ref_label_counts_host, components_host, nullptr, nullptr, 0, st,
                        &h->regions, h->named_nf > 0 ? h->named.data() : nullptr);
}

// ============================================================================= voice activity detection sweep
// tau_active trials of VoiceActivityDetection over a dataset: the speech curve of every chunk is computed once (vad_curve) and
// kept on the device; each trial then only thresholds it (vad_binarize).  Scoring merges every (file, trial)'s turns into
// whole-file segments and walks them against the file's speech reference with the DER kernels (der_components, M = 1, at
// most one reference label): with one label per side their false alarm and missed detection are DetectionErrorRate's.
struct dg_vad_sweep {
  int device = 0, F = 0, K = 0, nw = 1;
  int N = 0, nf = 0;                     // chunks and files of the curve; 0 until dg_vad_sweep_curve
  std::vector<int32_t> chunk_off;        // [nf + 1]
  DevBuf hamming, in, curve, header, turns, total, taus;
  DerBufs der;
  ScoredRegions regions;                 // dg_vad_sweep_set_scored_regions
  PinnedBuf pin;
};

extern "C" int dg_vad_sweep_create(int frames, int local_speakers, int num_windows, const double* hamming_host, int device,
                                   dg_vad_sweep** out) {
  if (!out || !hamming_host || frames < 1 || frames > 1023 || local_speakers < 1 || local_speakers > 64 || num_windows < 1 ||
      num_windows > 256) {
    set_error("dg_vad_sweep_create: need 1 <= frames <= 1023, 1 <= local_speakers <= 64, 1 <= num_windows <= 256");
    return DG_EINVAL;
  }
  DG_CUDA(cudaSetDevice(device));
  std::unique_ptr<dg_vad_sweep> h(new dg_vad_sweep());
  h->device = device; h->F = frames; h->K = local_speakers; h->nw = num_windows;
  if (h->hamming.ensure((size_t)frames * 8) || h->total.ensure(16)) return DG_ECUDA;
  DG_CUDA(cudaMemcpy(h->hamming.p, hamming_host, (size_t)frames * 8, cudaMemcpyHostToDevice));
  *out = h.release();
  return DG_OK;
}

extern "C" int dg_vad_sweep_destroy(dg_vad_sweep* h) {
  delete h;
  return DG_OK;
}

extern "C" int dg_vad_sweep_set_scored_regions(dg_vad_sweep* h, int num_files, const double* rows_host,
                                               const int32_t* offsets_host) {
  return set_scored_regions("dg_vad_sweep_set_scored_regions", h ? &h->regions : nullptr, num_files, rows_host,
                            offsets_host);
}

// The curve of Nv chunks with checked plan rows over the scores seg, chunk c being real chunk vchunk_host[c] of seg (null:
// chunk c); afterwards the handle's chunks and files are these, in nf files (file_off [nf + 1]).  Synchronises the stream.
static int vad_curve(dg_vad_sweep* h, const float* seg_dev, int Nv, const int32_t* plan_host, const int32_t* vchunk_host, int nf,
                     const int32_t* file_off, void* stream) {
  const int stride = 4 + h->nw;
  std::vector<long long> off(Nv + 1);
  off[0] = 0;
  for (int c = 0; c < Nv; c++) {
    const int32_t* pl = plan_host + (size_t)c * stride;
    off[c + 1] = off[c] + (pl[2] > 0 ? pl[2] : pl[1]);
  }
  DG_CUDA(cudaSetDevice(h->device));
  cudaStream_t st = (cudaStream_t)stream;
  // host -> device, one copy: curve offsets [Nv + 1] (int64, first: vad_binarize_all reads them there), plan [Nv][stride],
  // then with vchunk_host the chunk table [Nv]
  const size_t off_b = (size_t)(Nv + 1) * 8, plan_b = (size_t)Nv * stride * 4, vchunk_b = vchunk_host ? (size_t)Nv * 4 : 0;
  const size_t in_b = off_b + plan_b + vchunk_b;
  if (h->in.ensure(in_b) || h->curve.ensure((size_t)off[Nv] * 8) || h->pin.ensure(in_b)) return DG_ECUDA;
  unsigned char* pin = h->pin.as<unsigned char>();
  memcpy(pin, off.data(), off_b);
  memcpy(pin + off_b, plan_host, plan_b);
  if (vchunk_host) memcpy(pin + off_b + plan_b, vchunk_host, vchunk_b);
  unsigned char* din = h->in.as<unsigned char>();
  DG_CUDA(cudaMemcpyAsync(din, pin, in_b, cudaMemcpyHostToDevice, st));
  h->N = 0;   // no curve while it is being replaced
  int rc;
  if ((rc = launch_vad_curve_virtual(seg_dev, vchunk_host ? reinterpret_cast<const int32_t*>(din + off_b + plan_b) : nullptr, Nv,
                                     h->F, h->K, reinterpret_cast<const int32_t*>(din + off_b), stride, h->hamming.as<double>(),
                                     reinterpret_cast<const long long*>(din), h->curve.as<double>(), st)))
    return rc;
  DG_CUDA(cudaStreamSynchronize(st));
  h->N = Nv;
  h->nf = nf;
  h->chunk_off.assign(file_off, file_off + nf + 1);
  return DG_OK;
}

extern "C" int dg_vad_sweep_curve(dg_vad_sweep* h, const float* seg_dev, int N, int num_files,
                                  const int32_t* chunk_offsets_host, const int32_t* plan_host, void* stream) {
  const char* who = "dg_vad_sweep_curve";
  if (!h || !seg_dev || !plan_host || !chunk_offsets_host || N < 1 || num_files < 1) {
    set_error(std::string(who) + ": bad arguments (need N >= 1, num_files >= 1, non-null buffers)");
    return DG_EINVAL;
  }
  int rc;
  if ((rc = check_chunk_offsets(who, N, num_files, chunk_offsets_host)) ||
      (rc = check_file_plans(who, plan_host, num_files, chunk_offsets_host, h->nw, h->F)))
    return rc;
  return vad_curve(h, seg_dev, N, plan_host, nullptr, num_files, chunk_offsets_host, stream);
}

// The curve over the virtual layout of several latencies (check_virtual): the N real chunks of seg in units, the curve over the
// Nv virtual chunks.  Afterwards the handle's chunks and files are the virtual ones, so that dg_vad_sweep_run_files and
// dg_vad_sweep_score_files threshold and score every (latency, file) pair.
extern "C" int dg_vad_sweep_curve_latencies(dg_vad_sweep* h, const float* seg_dev, int N, int num_units,
                                            const int32_t* unit_offsets_host, int num_virtual, int num_virtual_files,
                                            const int32_t* vchunk_host, const int32_t* virtual_offsets_host,
                                            const int32_t* plan_host, void* stream) {
  const char* who = "dg_vad_sweep_curve_latencies";
  if (!h || !seg_dev) {
    set_error(std::string(who) + ": bad arguments (need a handle and scores)");
    return DG_EINVAL;
  }
  int rc;
  if ((rc = check_virtual(who, N, num_units, unit_offsets_host, num_virtual, num_virtual_files, vchunk_host,
                          virtual_offsets_host, plan_host, h->nw, h->F)))
    return rc;
  return vad_curve(h, seg_dev, num_virtual, plan_host, vchunk_host, num_virtual_files, virtual_offsets_host, stream);
}

// the argument checks of dg_vad_sweep_run_files / _score_files (before any launch)
static int vad_check(const char* who, dg_vad_sweep* h, const double* taus_host, int T) {
  if (!h || !taus_host || T < 1 || T > 65535) {
    set_error(std::string(who) + ": bad arguments (need 1 <= T <= 65535, non-null buffers)");
    return DG_EINVAL;
  }
  if (h->N < 1) {
    set_error(std::string(who) + ": no speech curve (dg_vad_sweep_curve first)");
    return DG_EINVAL;
  }
  if ((long long)h->nf * T > DG_SWEEP_MAX_STATES) {
    set_error(std::string(who) + ": " + std::to_string((long long)h->nf * T) + " (file, trial) states; at most " +
              std::to_string(DG_SWEEP_MAX_STATES) + " per call");
    return DG_EINVAL;
  }
  for (int t = 0; t < T; t++)
    if (!std::isfinite(taus_host[t])) {
      set_error(std::string(who) + ": the tau_active of trial " + std::to_string(t) + " is not finite");
      return DG_EINVAL;
    }
  return DG_OK;
}

// pinned layout of vad_binarize_all: taus [T] in; header [T][N][4], turn count, turn prefix out
static TurnOut vad_out(int T, int N) { return {(size_t)T * 8, (size_t)T * N * 16}; }

// the turns of T thresholds over the curve: header [T][N][4] and turns stay on the device, the count comes back in *total.
// with_header: the header and a turn prefix travel to the pinned buffer with the count (vad_out layout).  Synchronises `st`.
static int vad_binarize_all(dg_vad_sweep* h, const double* taus_host, int T, bool with_header, cudaStream_t st,
                            unsigned int* total_out) {
  const int N = h->N;
  const TurnOut lay = vad_out(T, N);
  const size_t turn_guess = std::max<size_t>((size_t)T * N * 4, (size_t)DG_POST_PREFIX);
  if (h->taus.ensure((size_t)T * 8) || h->header.ensure(lay.header_bytes) || h->turns.ensure(turn_guess * 4) ||
      h->pin.ensure(lay.end()))
    return DG_ECUDA;
  unsigned char* pin = h->pin.as<unsigned char>();
  memcpy(pin, taus_host, (size_t)T * 8);
  DG_CUDA(cudaMemcpyAsync(h->taus.p, pin, (size_t)T * 8, cudaMemcpyHostToDevice, st));
  const long long* d_off = reinterpret_cast<const long long*>(h->in.p);
  unsigned int total = 0;
  for (int attempt = 0; attempt < 2; attempt++) {
    const int cap = (int)std::min<size_t>(h->turns.bytes / 4, (size_t)INT32_MAX);
    DG_CUDA(cudaMemsetAsync(h->total.p, 0, 4, st));
    int rc;
    if ((rc = launch_vad_binarize(h->curve.as<double>(), d_off, N, T, h->taus.as<double>(), h->header.as<int32_t>(),
                                  h->turns.as<uint32_t>(), cap, h->total.as<unsigned int>(), st)))
      return rc;
    if (with_header) DG_CUDA(cudaMemcpyAsync(pin + lay.at, h->header.p, lay.header_bytes, cudaMemcpyDeviceToHost, st));
    DG_CUDA(cudaMemcpyAsync(pin + lay.total(), h->total.p, 4, cudaMemcpyDeviceToHost, st));
    if (with_header)
      DG_CUDA(cudaMemcpyAsync(pin + lay.prefix(), h->turns.p, (size_t)std::min(DG_POST_PREFIX, cap) * 4,
                              cudaMemcpyDeviceToHost, st));
    DG_CUDA(cudaStreamSynchronize(st));
    memcpy(&total, pin + lay.total(), 4);
    if (total <= (unsigned int)cap) break;
    // more turns than the device buffer holds: grow it to the count and binarise again
    if (h->turns.ensure((size_t)total * 4)) return DG_ECUDA;
  }
  *total_out = total;
  return DG_OK;
}

extern "C" int dg_vad_sweep_run_files(dg_vad_sweep* h, const double* taus_host, int T, int32_t* header_host,
                                      uint32_t* turns_host, int turn_cap_host, int* n_turns, void* stream) {
  const char* who = "dg_vad_sweep_run_files";
  int rc;
  if ((rc = vad_check(who, h, taus_host, T))) return rc;
  if (!header_host || !turns_host) {
    set_error(std::string(who) + ": bad arguments (need non-null header and turn buffers)");
    return DG_EINVAL;
  }
  DG_CUDA(cudaSetDevice(h->device));
  cudaStream_t st = (cudaStream_t)stream;
  unsigned int total = 0;
  if ((rc = vad_binarize_all(h, taus_host, T, true, st, &total))) return rc;
  return download_turns(who, h->pin.as<unsigned char>(), vad_out(T, h->N), h->turns.as<uint32_t>(), header_host, turns_host,
                        turn_cap_host, n_turns, st);
}

extern "C" int dg_vad_sweep_score_files(dg_vad_sweep* h, const double* taus_host, int T, const double* out_start_host,
                                        const double* out_res_host, const double* shifts_host, double collar,
                                        const double* ref_host, const int32_t* ref_offsets_host, double* components_host,
                                        void* stream) {
  const char* who = "dg_vad_sweep_score_files";
  int rc;
  if ((rc = vad_check(who, h, taus_host, T)) || (rc = regions_check(who, h->regions, h->nf))) return rc;
  const int N = h->N, nf = h->nf;
  if (!out_start_host || !out_res_host || !shifts_host || !components_host || !ref_offsets_host || !std::isfinite(collar) ||
      collar < 0) {
    set_error(std::string(who) + ": bad arguments (need chunk times, shifts, reference offsets, a components buffer, finite "
              "collar >= 0)");
    return DG_EINVAL;
  }
  for (int f = 0; f < nf; f++)
    if (!std::isfinite(shifts_host[f])) {
      set_error(std::string(who) + ": the shift of file " + std::to_string(f) + " is not finite");
      return DG_EINVAL;
    }
  for (int c = 0; c < N; c++)
    if (!std::isfinite(out_start_host[c]) || !std::isfinite(out_res_host[c])) {
      set_error(std::string(who) + ": chunk " + std::to_string(c) + " has an output time that is not finite");
      return DG_EINVAL;
    }
  if (ref_offsets_host[0] != 0) {
    set_error(std::string(who) + ": reference row offsets must start at 0");
    return DG_EINVAL;
  }
  for (int f = 0; f < nf; f++)
    if (ref_offsets_host[f + 1] < ref_offsets_host[f]) {
      set_error(std::string(who) + ": reference row offsets of file " + std::to_string(f) + " decrease");
      return DG_EINVAL;
    }
  const int S = ref_offsets_host[nf];
  if (S > 0 && !ref_host) {
    set_error(std::string(who) + ": non-null reference rows needed for " + std::to_string(S) + " rows");
    return DG_EINVAL;
  }
  // each file's reference is one label: its rows are a support (Timeline.support), finite, in time order, apart by more than
  // 1e-6 s (a gap that is a falsy Segment would have been merged)
  const std::vector<int32_t> labels((size_t)std::max(S, 1), 0);
  std::vector<int32_t> R(nf);
  for (int f = 0; f < nf; f++) {
    const int a = ref_offsets_host[f], n = ref_offsets_host[f + 1] - a;
    R[f] = n > 0 ? 1 : 0;
    if ((rc = sweep_check_reference(who, n > 0 ? ref_host + 2 * (size_t)a : nullptr, n > 0 ? labels.data() : nullptr, n, R[f])))
      return rc;
    for (int i = a + 1; i < a + n; i++)
      if (!(ref_host[2 * (size_t)i] - ref_host[2 * (size_t)i - 1] > 1e-6)) {
        set_error(std::string(who) + ": reference row " + std::to_string(i - a) + " of file " + std::to_string(f) +
                  " is not more than 1e-6 s after the previous one (the rows must be a support)");
        return DG_EINVAL;
      }
  }
  DG_CUDA(cudaSetDevice(h->device));
  cudaStream_t st = (cudaStream_t)stream;
  unsigned int total = 0;
  if ((rc = vad_binarize_all(h, taus_host, T, false, st, &total))) return rc;
  std::vector<double> comp((size_t)nf * T * 5);
  if ((rc = der_components(who, h->der, h->pin, h->header.as<int32_t>(), h->turns.as<uint32_t>(), total, N, nf,
                           h->chunk_off.data(), T, 1, out_start_host, out_res_host, shifts_host, collar, ref_host,
                           labels.data(), ref_offsets_host, R.data(), comp.data(), nullptr, nullptr, 0, st, &h->regions)))
    return rc;
  for (size_t i = 0; i < (size_t)nf * T; i++) {
    components_host[2 * i] = comp[5 * i];           // false alarm
    components_host[2 * i + 1] = comp[5 * i + 1];   // missed detection
  }
  return DG_OK;
}
