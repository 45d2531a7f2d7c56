// Many live audio streams on one device (dg_multi_*): the reference's live loop (inference.py: one window per stream every
// step, SpeakerDiarization.__call__ with a batch of one, diarization.py:172-232) for up to `slots` streams at once, batched
// across the streams.  Work happens in ticks: every open stream contributes its complete, unconsumed windows (at most
// max_wps), and those windows run as ONE batch -- one upload, one network pass (in sub-batches on the two scratch lanes),
// one clustering launch with a state per stream, one post-path launch with a history per stream, one download.  Each stream
// may have its own latency (num_windows, up to the handle's) and {tau, rho, delta} (dg_multi_open_config): none of them
// reaches the networks, so the clustering runs each state at its stream's row and the post-path each chunk at its stream's.
//
// A VAD handle (dg_multi_create_vad) serves the reference's VoiceActivityDetection the same way: the same audio in, the
// segmentation network alone, and per stream its speech curve (max over the local speakers) aggregated and binarised on the
// device, with a history of max curves per stream.  It has no embedding model and no clustering state.
#include <string.h>

#include <algorithm>
#include <cmath>
#include <map>
#include <memory>
#include <vector>

#include "host.cuh"

// The windows of a source rate: S and hop source samples per window / between windows, ring capacity `cap` (what a stream may
// hold unconsumed).  A declared rate (g.o > 0) resamples each window to the pipeline's chunk (taps of rs): g is its geometry, a hop is
// fs whole 16 kHz frames, frames r_lo .. r_hi of a window have all their taps inside it, and the slot's 16 kHz ring holds Q
// frames -- the interior frames of max_wps consecutive windows.
struct RateGeom {
  int S = 0, hop = 1, cap = 0;
  const dg_resample* rs = nullptr;
  RsGeom g{};
  long long fs = 0, r_lo = 0, r_hi = -1, Q = 0;
  bool resampled() const { return g.o > 0; }
};

static long long ring_capacity(long long S, long long hop, int max_wps) { return (S + 2LL * max_wps * hop + 1023) / 1024 * 1024; }

// the geometry of a source rate resampled by g to windows of out_S samples, or DG_EINVAL naming what rules it out
static int rate_geom(const RsGeom& g, int S, int hop, int out_S, int max_wps, RateGeom& r, const char* who) {
  if (S < 1 || hop < 1 || hop > S) {
    set_error(std::string(who) + ": chunk and step must be positive, step <= chunk");
    return DG_EINVAL;
  }
  if (resample_out_len(g, S) != out_S) {
    set_error(std::string(who) + ": a chunk of " + std::to_string(S) + " source samples resamples to " +
              std::to_string(resample_out_len(g, S)) + " samples, not the pipeline's " + std::to_string(out_S));
    return DG_EINVAL;
  }
  if (hop % g.o) {
    set_error(std::string(who) + ": a step of " + std::to_string(hop) + " source samples is not a whole number of frames (" +
              std::to_string(g.o) + " samples each)");
    return DG_EINVAL;
  }
  r = RateGeom{};
  r.S = S;
  r.hop = hop;
  r.g = g;
  r.fs = hop / g.o;
  r.r_lo = (g.w + g.o - 1) / g.o;
  r.r_hi = S - g.w - g.o >= 0 ? (S - g.w - g.o) / g.o : -1;
  r.Q = (max_wps - 1) * r.fs + std::max(0LL, r.r_hi - r.r_lo + 1);
  const long long cap = ring_capacity(S, hop, max_wps);
  if (cap > (1 << 30) || r.Q * g.n > (1 << 30)) {
    set_error(std::string(who) + ": the rings of this rate exceed 2^30 samples per stream");
    return DG_EINVAL;
  }
  r.cap = (int)cap;
  return DG_OK;
}

// What a tick does besides the networks: its slots and rows (all B rows, and the rows at the pipeline's rate with their window
// starts), and per declared rate the resampling items and the resampled rows, grouped by rate (entries [off[i], off[i + 1])
// belong to rate 1 + i); done[a]: frames of act[a]'s stream computed once the tick has run.
struct TickPlan {
  std::vector<TickSlot> act;
  int B = 0;
  std::vector<int2> rows, rows16;
  std::vector<long long> start, start16;
  std::vector<RsFrames> items;
  std::vector<RsRow> rs_rows;
  std::vector<int> item_off, row_off;
  std::vector<long long> done;
};

// the pipeline's own rate: a ring with room for the windows of a tick and as much audio again pushed ahead (as dg_stream)
static RateGeom pipeline_rate(int S, int hop, int max_wps) {
  RateGeom r;
  r.S = S;
  r.hop = hop;
  r.cap = (int)ring_capacity(S, hop, max_wps);
  return r;
}

// The audio of the stream in a slot: its rate (index into SlotBook::rates), whether the slot is open, and the absolute sample
// counters pushed (staged included) / start of the next window, and for a resampled stream the 16 kHz frames computed so far.
struct SlotAudio {
  int rate = 0;
  bool open = false;
  long long wpos = 0, rpos = 0, done = 0;
};

// The host bookkeeping of the streams' audio, no device work: a SlotAudio per slot; the samples pushed since the last tick
// are [0, n_staged) of a staging buffer, described by `pieces` in push order.  A piece is a run of ONE slot's samples that is
// contiguous both in the staging buffer and in that slot's stream, so a piece is extended only by a push that continues it
// in both.  Every slot's ring has stride C (the largest capacity of any rate).
struct SlotBook {
  int C = 0;
  std::vector<RateGeom> rates;                // [0]: the pipeline's rate; [1 + id]: declared rate id
  std::vector<SlotAudio> audio;
  std::vector<RingPiece> pieces;
  long long n_staged = 0;

  void init(int slots, const RateGeom& base) {
    rates.assign(1, base);
    C = base.cap;
    audio.assign(slots, SlotAudio{});
  }
  void add_rate(const RateGeom& r) {
    rates.push_back(r);
    C = std::max(C, r.cap);
  }
  bool ok(int slot) const { return slot >= 0 && slot < (int)audio.size() && audio[slot].open; }
  const RateGeom& geom(int s) const { return rates[audio[s].rate]; }
  long long available(int s) const {    // complete windows, pushed and not consumed
    const RateGeom& r = geom(s);
    const long long have = audio[s].wpos - audio[s].rpos;
    return have < r.S ? 0 : (have - r.S) / r.hop + 1;
  }
  // a stream starts in `slot` at a's rate and counters (a new stream: all zero)
  void start(int slot, SlotAudio a = {}) {
    a.open = true;
    audio[slot] = a;
  }
  // the stream ends: its staged samples are dropped (they stay in the staging buffer, no piece refers to them)
  void stop(int slot) {
    audio[slot].open = false;
    pieces.erase(std::remove_if(pieces.begin(), pieces.end(), [&](const RingPiece& p) { return p.slot == slot; }),
                 pieces.end());
  }
  bool fits(int slot, int n) const { return audio[slot].wpos + n - audio[slot].rpos <= geom(slot).cap; }
  // books n > 0 samples of `slot` at staging offset n_staged (the caller copies them there)
  void push(int slot, int n) {
    RingPiece* last = pieces.empty() ? nullptr : &pieces.back();
    if (last && last->slot == slot && last->src + last->n == n_staged && last->dst + last->n == audio[slot].wpos)
      last->n += n;
    else
      pieces.push_back(RingPiece{n_staged, audio[slot].wpos, slot, n});
    n_staged += n;
    audio[slot].wpos += n;
  }
  void uploaded() {
    pieces.clear();
    n_staged = 0;
  }
  // the tick's plan: every open slot with windows gives up to max_wps, in slot order.  A resampled stream's item is the frames
  // its windows' interiors need that no earlier tick computed: [max(done, first start / o + r_lo), last start / o + r_hi]
  void plan(int max_wps, TickPlan& t) const {
    t = TickPlan{};
    const int nr = (int)rates.size();
    std::vector<std::vector<RsFrames>> items(nr);
    std::vector<std::vector<RsRow>> rs_rows(nr);
    for (int s = 0; s < (int)audio.size(); s++) {
      const SlotAudio& a = audio[s];
      const int n = a.open ? (int)std::min<long long>(available(s), max_wps) : 0;
      if (!n) continue;
      const RateGeom& r = geom(s);
      t.act.push_back(TickSlot{s, t.B, n, 0, 0, 1, {0, 0}});
      long long d = a.done;
      for (int i = 0; i < n; i++) {
        const long long st = a.rpos + (long long)i * r.hop;
        t.rows.push_back(make_int2((int)t.act.size() - 1, i));
        t.start.push_back(st);
        if (r.resampled())
          rs_rows[a.rate].push_back(RsRow{st, st / r.g.o, s, t.B + i});
      }
      if (r.resampled()) {
        const long long lo = std::max(d, a.rpos / r.g.o + r.r_lo);
        const long long hi = (a.rpos + (long long)(n - 1) * r.hop) / r.g.o + r.r_hi;
        if (hi >= lo) {
          items[a.rate].push_back(RsFrames{lo, s, (int)(hi - lo + 1)});
          d = hi + 1;
        }
      }
      t.done.push_back(d);
      t.B += n;
    }
    for (int b = 0; b < t.B; b++)
      if (!geom(t.act[t.rows[b].x].slot).resampled()) {
        t.rows16.push_back(t.rows[b]);
        t.start16.push_back(t.start[b]);
      }
    t.item_off.assign(1, 0);
    t.row_off.assign(1, 0);
    for (int i = 1; i < nr; i++) {
      t.items.insert(t.items.end(), items[i].begin(), items[i].end());
      t.rs_rows.insert(t.rs_rows.end(), rs_rows[i].begin(), rs_rows[i].end());
      t.item_off.push_back((int)t.items.size());
      t.row_off.push_back((int)t.rs_rows.size());
    }
  }
  // the tick of plan t has run: its windows are consumed and its frames computed
  void consumed(const TickPlan& t) {
    for (size_t a = 0; a < t.act.size(); a++) {
      const int s = t.act[a].slot;
      audio[s].rpos += (long long)t.act[a].n * geom(s).hop;
      audio[s].done = t.done[a];
    }
  }
};

// The values of the stream in a slot besides its audio (SlotAudio): its latency / step nw (<= the handle's), post-path
// history entries and current copy, {tau, rho, delta} (a VAD handle: {tau, 0, 0}), the gallery and threshold it is named from
// (null: none), whether it has had a tick, and its named global speakers (bit g; the host mirror of the device's table).
struct SlotStream {
  int nw = 1, n_hist = 0, cur = 0;
  double par[3] = {0.0, 0.0, 0.0};
  dg_gallery* gal = nullptr;
  double thr = 0.0;
  bool ticked = false;
  uint32_t named = 0;
};

struct dg_multi {
  int device = 0, slots = 0, max_wps = 0;
  int S = 0, hop = 0;                         // samples per window, between windows
  int F = 0, K = 0, D = 0, M = 0, nw = 1;     // nw: the largest latency / step of any stream (sizes the histories)
  double tau = 0.5, rho = 0.3, delta = 1.0;   // the values of a stream opened without its own
  NetLanes net;
  SlotBook book;
  std::vector<SlotStream> streams;            // per slot
  PinnedBuf stage;                            // staged samples [0, book.n_staged), then a tick's tables
  DevBuf yrings;                              // resampled streams: 16 kHz rings [slots][Y]
  long long Y = 0;
  bool opened = false;                        // a stream was opened (rates can no longer be added)
  int last_B = 0;                             // windows of the last tick that had any
  DevBuf rings, hamming, in, wav, seg, emb, maps, centers, active, init, prep, prep_d, hist_seg, hist_map, header, turns, total;
  DevBuf hist_vad;                            // VAD mode (net.emb null): per slot the last nw - 1 max curves [2][slots][nw - 1][F]
  PinnedBuf pin_out;                          // header, turn count and turn prefix of a tick (TurnOut layout at 0)
  Stream st;
  Event e_start, e_lane_done[2];
  Event t_begin, t_end;                       // timing events around the last tick's device work on `st`
  bool timed = false;                         // a tick has run
  // gallery naming: the default gallery and threshold of every stream (dg_multi_set_gallery).  Once the handle has received a
  // gallery (naming): per slot the named global speakers (bit g) and their claimed entries [slots][32], indices into the
  // slot's gallery, on the device (the named bits mirrored in SlotStream::named); a tick's queries, segments, query offset
  // and count per group, split partials and new names {slot, g, entry}
  dg_gallery* gal = nullptr;
  double gal_threshold = 0.0;
  bool naming = false;
  DevBuf gal_named, gal_claimed, gal_q, gal_seg, gal_gq, gal_d, gal_e, gal_list;
  std::vector<int32_t> names_last;            // the names the last dg_multi_step decided, [n][3]
  // dg_multi_export / dg_multi_import: one round's packed states and its piece list, on the device and pinned.  Allocated
  // by the first move that needs them (a growth synchronises the device, as every DevBuf growth does) and kept for the
  // handle's life: at most XFER_STAGING bytes of states plus the pieces, each.
  DevBuf xfer;
  PinnedBuf xfer_pin;
};

// In front of the header in h->header and in the tick's pinned download, once the handle has received a gallery: the count
// of the tick's new names (16 bytes) and the first GAL_NAME_PREFIX of them, so that they travel in the header's copy
static size_t names_bytes(const dg_multi* h) { return h->naming ? 16 + (size_t)GAL_NAME_PREFIX * 12 : 0; }

// The grouped gallery search of a tick (gallery_plan): groups (one per distinct gallery and threshold, in order of their
// first slot), the tick's slots with a gallery as segments {slot, group} (group by group, slots in order), the work list,
// the upper bound of the queries and the largest split count.
struct GalTick {
  std::vector<GalGroup> groups;
  std::vector<int> keys;        // the gallery key of each group
  std::vector<int2> segs;
  std::vector<GalWork> work;
  int queries = 0, splits = 0;
};

// the plan of n slots in slot order: slot[a], its gallery key[a] (-1: none; keys index G / thr), its unnamed speakers
// unnamed[a]; the groups' gallery pointers are left null
static void gallery_tick_plan(const int* slot, const int* key, const int* unnamed, int n, const int* G, const double* thr,
                              GalTick& t) {
  t = GalTick{};
  std::vector<int> group_of_key;
  std::vector<int>& keys = t.keys;
  for (int a = 0; a < n; a++) {
    const int k = key[a];
    if (k < 0) continue;
    if (k >= (int)group_of_key.size()) group_of_key.resize(k + 1, -1);
    if (group_of_key[k] < 0) {
      group_of_key[k] = (int)keys.size();
      keys.push_back(k);
    }
  }
  // the segments bucketed by group in one pass (a counting sort, stable in slot order): O(slots + groups)
  const int ng = (int)keys.size();
  t.groups.resize(ng);
  std::vector<int> fill(ng + 1, 0);
  for (int a = 0; a < n; a++)
    if (key[a] >= 0) fill[group_of_key[key[a]] + 1]++;
  for (int r = 0; r < ng; r++) fill[r + 1] += fill[r];
  for (int r = 0; r < ng; r++)
    t.groups[r] = GalGroup{nullptr, nullptr, thr[keys[r]], G[keys[r]], 0, 0, 0, 0, fill[r], fill[r + 1], 0};
  t.segs.resize(fill[ng]);
  for (int a = 0; a < n; a++) {
    if (key[a] < 0) continue;
    const int r = group_of_key[key[a]];
    t.segs[fill[r]++] = make_int2(slot[a], r);
    t.groups[r].q_ub += unnamed[a];
    t.queries += unnamed[a];
  }
  t.splits = gallery_plan(t.groups, t.work);
}

static bool slot_ok(const dg_multi* h, int slot) { return h && h->book.ok(slot); }
static bool vad_mode(const dg_multi* h) { return !h->net.emb; }

// The host side of a handle, no device work: `slots` slots, all closed, taking up to max_wps windows of S samples every hop
// at the pipeline's rate, of F frames and K local speakers, aggregating up to nw buffers
static void multi_init(dg_multi& h, int device, int slots, int max_wps, int S, int hop, int F, int K, int nw) {
  h.device = device; h.slots = slots; h.max_wps = max_wps;
  h.S = S; h.hop = hop; h.F = F; h.K = K; h.nw = nw;
  h.book.init(slots, pipeline_rate(S, hop, max_wps));
  h.streams.assign(slots, SlotStream{});
}

// The device side of a handle set up by multi_init (its mode, M and D set): the rings, the Hamming window, the histories and
// (diarization) clustering states of every slot, the scratch lanes, stream and events.  On success *out owns the handle.
static int multi_alloc(std::unique_ptr<dg_multi> h, const double* hamming_host, dg_multi** out) {
  const size_t n = (size_t)h->slots, hist = (size_t)std::max(1, h->nw - 1), F = (size_t)h->F, K = (size_t)h->K;
  DG_CUDA(cudaSetDevice(h->device));
  if (h->rings.ensure(n * h->book.C * 4) || h->hamming.ensure(F * 8) || h->total.ensure(16)) return DG_ECUDA;
  if (vad_mode(h.get()) ? h->hist_vad.ensure(2 * n * hist * F * 4)
                        : (h->centers.ensure(n * h->M * h->D * 8) || h->active.ensure(n * 32 * 4) || h->init.ensure(n * 2 * 4) ||
                           h->hist_seg.ensure(2 * n * hist * F * K * 4) || h->hist_map.ensure(2 * n * hist * K * 4)))
    return DG_ECUDA;
  DG_CUDA(cudaMemcpy(h->hamming.p, hamming_host, F * 8, cudaMemcpyHostToDevice));
  if (net_lanes_create(h->net) || h->st.create() || h->e_start.create() || h->e_lane_done[0].create() ||
      h->e_lane_done[1].create() || h->t_begin.create(cudaEventDefault) || h->t_end.create(cudaEventDefault))
    return DG_ECUDA;
  *out = h.release();
  return DG_OK;
}

extern "C" int dg_multi_create(dg_seg* seg, dg_emb* emb, int chunk_samples, int step_samples, int max_streams,
                               int max_windows_per_stream, int max_speakers, double tau, double rho, double delta, float gamma,
                               float beta, int normalize_weights, int num_windows, const double* hamming_host, dg_multi** out) {
  if (!seg || !emb || !out || !hamming_host) {
    set_error("dg_multi_create: null handle or buffer");
    return DG_EINVAL;
  }
  if (seg->device != emb->device) {
    set_error("dg_multi_create: handles live on different devices");
    return DG_EINVAL;
  }
  if (chunk_samples < 4 || step_samples < 4 || chunk_samples % 4 || step_samples % 4 || step_samples > chunk_samples) {
    set_error("dg_multi_create: chunk and step must be positive multiples of 4 samples, step <= chunk");
    return DG_EINVAL;
  }
  if (max_streams < 1 || max_windows_per_stream < 1 || (long long)max_streams * max_windows_per_stream > 65535 ||
      num_windows < 1 || num_windows > 256 || max_speakers < 1 || max_speakers > 32 || !std::isfinite(tau) || !std::isfinite(rho) ||
      !std::isfinite(delta)) {
    set_error("dg_multi_create: need max_streams, max_windows_per_stream >= 1 with a product <= 65535, 1 <= num_windows "
              "<= 256, 1 <= max_speakers <= 32 and finite thresholds");
    return DG_EINVAL;
  }
  int rc, F = 0, K = 0;
  if ((rc = dg_seg_dims(seg, chunk_samples, &F, &K))) return rc;
  const int D = emb->D;
  const size_t cluster_smem = ((size_t)max_speakers * D + (size_t)K * D) * 8 + (size_t)2 * K * D * 4;
  if (K > 8 || K > max_speakers || F > 1023 || cluster_smem > 200 * 1024) {
    set_error("dg_multi_create: need local speakers <= min(8, max_speakers), frames <= 1023 and a centroid table of at most "
              "200 KB");
    return DG_EINVAL;
  }
  std::unique_ptr<dg_multi> h(new dg_multi());
  multi_init(*h, seg->device, max_streams, max_windows_per_stream, chunk_samples, step_samples, F, K, num_windows);
  h->D = D; h->M = max_speakers;
  h->tau = tau; h->rho = rho; h->delta = delta;
  h->net.seg = seg; h->net.emb = emb;
  h->net.gamma = gamma; h->net.beta = beta; h->net.normalize_weights = normalize_weights;
  return multi_alloc(std::move(h), hamming_host, out);
}

// The numbers are checked before the handles, so that every refusal can be seen without a device.
extern "C" int dg_multi_create_vad(dg_seg* seg, int chunk_samples, int step_samples, int max_streams, int max_windows_per_stream,
                                   double tau, int num_windows, const double* hamming_host, dg_multi** out) {
  if (chunk_samples < 4 || step_samples < 4 || chunk_samples % 4 || step_samples % 4 || step_samples > chunk_samples) {
    set_error("dg_multi_create_vad: chunk and step must be positive multiples of 4 samples, step <= chunk");
    return DG_EINVAL;
  }
  if (max_streams < 1 || max_windows_per_stream < 1 || (long long)max_streams * max_windows_per_stream > 65535 ||
      num_windows < 1 || num_windows > 256 || !std::isfinite(tau)) {
    set_error("dg_multi_create_vad: need max_streams, max_windows_per_stream >= 1 with a product <= 65535, 1 <= num_windows "
              "<= 256 and a finite threshold");
    return DG_EINVAL;
  }
  if (!seg || !out || !hamming_host) {
    set_error("dg_multi_create_vad: null handle or buffer");
    return DG_EINVAL;
  }
  int rc, F = 0, K = 0;
  if ((rc = dg_seg_dims(seg, chunk_samples, &F, &K))) return rc;
  if (K > 8 || F > 1023) {
    set_error("dg_multi_create_vad: need local speakers <= 8 and frames <= 1023");
    return DG_EINVAL;
  }
  std::unique_ptr<dg_multi> h(new dg_multi());
  multi_init(*h, seg->device, max_streams, max_windows_per_stream, chunk_samples, step_samples, F, K, num_windows);
  h->M = 1;   // one "speaker": speech
  h->tau = tau;
  h->net.seg = seg;
  return multi_alloc(std::move(h), hamming_host, out);
}

extern "C" int dg_multi_destroy(dg_multi* h) {
  delete h;
  return DG_OK;
}

// a source rate whose windows `rs` resamples to the pipeline's chunk; before any stream is opened (the rings grow)
extern "C" int dg_multi_add_rate(dg_multi* h, dg_resample* rs, int chunk_samples, int step_samples, int* rate_id) {
  const char* who = "dg_multi_add_rate";
  if (!h || !rs || !rate_id) {
    set_error(std::string(who) + ": null handle");
    return DG_EINVAL;
  }
  if (h->opened) {
    set_error(std::string(who) + ": rates are added before any stream is opened");
    return DG_EINVAL;
  }
  if (rs->device != h->device) {
    set_error(std::string(who) + ": the resampler lives on another device");
    return DG_EINVAL;
  }
  for (size_t i = 1; i < h->book.rates.size(); i++)
    if (h->book.rates[i].g.o == rs->g.o && h->book.rates[i].g.n == rs->g.n) {
      set_error(std::string(who) + ": this rate was added before (rate id " + std::to_string(i - 1) + ")");
      return DG_EINVAL;
    }
  RateGeom r;
  int rc;
  if ((rc = rate_geom(rs->g, chunk_samples, step_samples, h->S, h->max_wps, r, who))) return rc;
  r.rs = rs;
  DG_CUDA(cudaSetDevice(h->device));
  const int C = std::max(h->book.C, r.cap);
  const long long Y = std::max(h->Y, r.Q * r.g.n);
  if (h->rings.ensure((size_t)h->slots * C * 4) || h->yrings.ensure((size_t)h->slots * Y * 4)) return DG_ECUDA;
  h->book.add_rate(r);
  h->Y = Y;
  *rate_id = (int)h->book.rates.size() - 2;
  return DG_OK;
}

// The host bookkeeping of a stream that starts in `slot` (closed) with values x and audio a (a new stream: fresh values and
// zero counters at its rate; a restored one: what it had)
static void stream_begin(dg_multi* h, int slot, const SlotStream& x, const SlotAudio& a) {
  h->book.start(slot, a);
  h->streams[slot] = x;
  h->opened = true;
}

// the stream in open `slot` ends: its staged samples are dropped, and the handle no longer refers to its gallery
static void stream_end(dg_multi* h, int slot) {
  h->book.stop(slot);
  h->streams[slot].gal = nullptr;
}

// slots [s0, s0 + n) with nothing named or claimed, on the device (on h->st) and in the host mirror; the tables exist
static int clear_names(dg_multi* h, int s0, int n) {
  DG_CUDA(cudaMemsetAsync(h->gal_named.as<uint32_t>() + s0, 0, (size_t)n * 4, h->st));
  DG_CUDA(cudaMemsetAsync(h->gal_claimed.as<int32_t>() + (size_t)s0 * 32, 0xff, (size_t)n * 32 * 4, h->st));
  for (int s = s0; s < s0 + n; s++) h->streams[s].named = 0;
  return DG_OK;
}

// a new stream in `slot` at declared rate `rate_id` (-1: the pipeline's rate), aggregating num_windows buffers, with
// params {tau, rho, delta} (a VAD handle reads tau only): empty rings, no history, and the clustering state (a VAD handle has
// none) fresh (the reference's SpeakerDiarization.reset()) for n = 0, else seeded with the n known centroids centers_host
// [n][D]: rows 0 .. n - 1 written and active, the rest zero, initialised.  Every argument is checked first; a refusal names
// `who` and changes nothing.
static int open_slot(dg_multi* h, int slot, int rate_id, int num_windows, const double* params, const double* centers_host,
                     int n, const char* who) {
  if (!h || slot < 0 || slot >= h->slots || h->book.audio[slot].open) {
    set_error(std::string(who) + ": slot " + std::to_string(slot) + " is out of range or already open");
    return DG_EINVAL;
  }
  if (rate_id < -1 || rate_id + 1 >= (int)h->book.rates.size()) {
    set_error(std::string(who) + ": rate " + std::to_string(rate_id) + " was not declared");
    return DG_EINVAL;
  }
  if (num_windows < 1 || num_windows > h->nw) {
    set_error(std::string(who) + ": num_windows " + std::to_string(num_windows) + " is outside [1, " + std::to_string(h->nw) +
              "], the handle's maximum");
    return DG_EINVAL;
  }
  const bool vad = vad_mode(h);
  if (!params || !std::isfinite(params[0]) || (!vad && (!std::isfinite(params[1]) || !std::isfinite(params[2])))) {
    set_error(std::string(who) + (vad ? ": need a finite tau" : ": need finite tau, rho and delta"));
    return DG_EINVAL;
  }
  if (n < 0 || n > h->M || (n > 0 && (vad || !centers_host))) {
    set_error(std::string(who) + ": need 0 <= n <= max_speakers (" + std::to_string(h->M) + ") known centroids and a "
              "non-null table, got n = " + std::to_string(n));
    return DG_EINVAL;
  }
  const int D = h->D;
  for (int i = 0; i < n; i++) {
    double ss = 0.0;
    bool finite = true;
    for (int d = 0; d < D; d++) {
      const double x = centers_host[(size_t)i * D + d];
      finite = finite && std::isfinite(x);
      ss += x * x;
    }
    if (!finite || !(ss > 0.0)) {
      set_error(std::string(who) + ": centroid " + std::to_string(i) + (finite ? " has a zero norm" : " is not finite"));
      return DG_EINVAL;
    }
  }
  DG_CUDA(cudaSetDevice(h->device));
  const size_t s = (size_t)slot;
  if (!vad) {
    double* centers = h->centers.as<double>() + s * h->M * D;
    DG_CUDA(cudaMemsetAsync(centers, 0, (size_t)h->M * D * 8, h->st));
    DG_CUDA(cudaMemsetAsync(h->active.as<int>() + s * 32, 0, 32 * 4, h->st));
    DG_CUDA(cudaMemsetAsync(h->init.as<int>() + s * 2, 0, 2 * 4, h->st));
    if (n > 0) {
      // copies from pageable memory: the source is staged before cudaMemcpyAsync returns, so it may be freed then
      const std::vector<int> flags((size_t)n, 1);
      const int init[2] = {1, 0};
      DG_CUDA(cudaMemcpyAsync(centers, centers_host, (size_t)n * D * 8, cudaMemcpyHostToDevice, h->st));
      DG_CUDA(cudaMemcpyAsync(h->active.as<int>() + s * 32, flags.data(), (size_t)n * 4, cudaMemcpyHostToDevice, h->st));
      DG_CUDA(cudaMemcpyAsync(h->init.as<int>() + s * 2, init, 2 * 4, cudaMemcpyHostToDevice, h->st));
    }
  }
  int rc;
  if (h->naming && (rc = clear_names(h, slot, 1))) return rc;   // a stream opens with no speaker named
  SlotStream x{num_windows, 0, 0, {params[0], vad ? 0.0 : params[1], vad ? 0.0 : params[2]}};
  if (!vad) {   // named from the default gallery unless dg_multi_set_slot_gallery gives it its own
    x.gal = h->gal;
    x.thr = h->gal_threshold;
  }
  stream_begin(h, slot, x, SlotAudio{rate_id + 1});
  return DG_OK;
}

extern "C" int dg_multi_open_config(dg_multi* h, int slot, int rate_id, int num_windows, const double* params) {
  return open_slot(h, slot, rate_id, num_windows, params, nullptr, 0, "dg_multi_open_config");
}

extern "C" int dg_multi_open_seeded(dg_multi* h, int slot, int rate_id, int num_windows, const double* params,
                                    const double* centers_host, int n) {
  if (h && vad_mode(h)) {
    set_error("dg_multi_open_seeded: a VAD handle has no clustering state to seed");
    return DG_EINVAL;
  }
  return open_slot(h, slot, rate_id, num_windows, params, centers_host, n, "dg_multi_open_seeded");
}

extern "C" int dg_multi_open_rate(dg_multi* h, int slot, int rate_id) {
  if (!h) {
    set_error("dg_multi_open: null handle");
    return DG_EINVAL;
  }
  const double params[3] = {h->tau, h->rho, h->delta};
  return open_slot(h, slot, rate_id, h->nw, params, nullptr, 0, "dg_multi_open");
}

extern "C" int dg_multi_open(dg_multi* h, int slot) { return dg_multi_open_rate(h, slot, -1); }

// the stream in `slot` ends: its staged samples are dropped, the slot can be opened again
extern "C" int dg_multi_close(dg_multi* h, int slot) {
  if (!slot_ok(h, slot)) {
    set_error("dg_multi_close: slot " + std::to_string(slot) + " is not open");
    return DG_EINVAL;
  }
  stream_end(h, slot);
  return DG_OK;
}

// the clustering state of the open stream in `slot` after the last tick: centroids [M][D], active flags [M], initialised
extern "C" int dg_multi_get_state(dg_multi* h, int slot, double* centers_host, int32_t* active_host, int* initialized) {
  if (!slot_ok(h, slot) || vad_mode(h) || !centers_host || !active_host || !initialized) {
    set_error("dg_multi_get_state: need an open slot of a diarization handle and non-null outputs");
    return DG_EINVAL;
  }
  DG_CUDA(cudaSetDevice(h->device));
  const size_t s = (size_t)slot;
  int init[2] = {0, 0};
  DG_CUDA(cudaMemcpyAsync(centers_host, h->centers.as<double>() + s * h->M * h->D, (size_t)h->M * h->D * 8,
                          cudaMemcpyDeviceToHost, h->st));
  DG_CUDA(cudaMemcpyAsync(active_host, h->active.as<int>() + s * 32, (size_t)h->M * 4, cudaMemcpyDeviceToHost, h->st));
  DG_CUDA(cudaMemcpyAsync(init, h->init.as<int>() + s * 2, 2 * 4, cudaMemcpyDeviceToHost, h->st));
  DG_CUDA(cudaStreamSynchronize(h->st));
  if (init[1]) {
    set_error("Cannot update unknown centers");   // reference clustering.py:98 (AssertionError)
    return DG_EINVAL;
  }
  *initialized = init[0];
  return DG_OK;
}

extern "C" int dg_multi_available(const dg_multi* h, int slot) {
  if (!slot_ok(h, slot)) {
    set_error("dg_multi_available: slot " + std::to_string(slot) + " is not open");
    return DG_EINVAL;
  }
  return (int)h->book.available(slot);
}

// appends n samples to the stream in `slot`: copied into the pinned staging, uploaded at the next dg_multi_step
extern "C" int dg_multi_push_host(dg_multi* h, int slot, const float* samples, int n) {
  if (!slot_ok(h, slot) || n < 0 || (n > 0 && !samples)) {
    set_error("dg_multi_push_host: bad arguments (an open slot, n >= 0 samples)");
    return DG_EINVAL;
  }
  if (!h->book.fits(slot, n)) {
    set_error("dg_multi_push_host: ring of slot " + std::to_string(slot) + " full (" +
              std::to_string(h->book.audio[slot].wpos - h->book.audio[slot].rpos) + " samples buffered, capacity " +
              std::to_string(h->book.geom(slot).cap) + "): step first");
    return DG_EINVAL;
  }
  if (n == 0) return DG_OK;
  const long long staged = h->book.n_staged;
  const size_t need = (size_t)(staged + n) * 4;
  if (need > h->stage.bytes) {   // grow, keeping what is staged (no upload reads the staging between ticks)
    PinnedBuf bigger;
    if (bigger.ensure(std::max(need, 2 * h->stage.bytes))) return DG_ECUDA;
    if (staged) memcpy(bigger.h, h->stage.h, (size_t)staged * 4);
    h->stage = std::move(bigger);
  }
  memcpy(h->stage.as<float>() + staged, samples, (size_t)n * 4);
  h->book.push(slot, n);
  return DG_OK;
}

static size_t align16(size_t b) { return (b + 15) & ~(size_t)15; }

// Where the tables of a tick lie in its one host -> device copy (byte offsets into h->in): staged samples at 0, pieces [np],
// slots [n_act], rows [B] {slot entry, window}, window starts [B], plan [B][stride], cluster states [n_act] {slot, entry},
// chunk offsets [slots + 1] by slot (states and offsets are read by a diarization tick only), thresholds [n_act][3] {tau, rho,
// delta} of each slot entry.  A tick with resampled rows also carries the rows at the pipeline's rate [n16] with their starts,
// the resampling items and the resampled rows.
struct TickIn {
  size_t o_pieces, o_act, o_rows, o_start, o_plan, o_states, o_off, o_trials, o_rows16, o_start16, o_items, o_rs, bytes;
  size_t o_groups, o_segs, o_work;   // with gallery queries: the groups, segments and work list of the grouped search
  bool mixed;
};

// The audio-in half of a tick, the same in both modes: ONE copy of the staged samples and the tick's tables to h->in (t_begin
// recorded before it), the staged samples to their rings, then the batch [B, S] of windows to h->wav, grouped by slot (windows
// at a declared rate resampled); e_start marks the batch complete on h->st.  A tick with gallery queries (gt) carries the
// plan of its grouped search after the other tables.
static int tick_audio_in(dg_multi* h, const TickPlan& tp, const int32_t* plan_host, const GalTick* gt, TickIn& L) {
  cudaStream_t st = h->st;
  const std::vector<TickSlot>& act = tp.act;
  const int B = tp.B, n_act = (int)act.size(), np = (int)h->book.pieces.size(), S = h->S, stride = 4 + h->nw;
  L.o_pieces = align16((size_t)h->book.n_staged * 4);
  L.o_act = L.o_pieces + align16((size_t)np * sizeof(RingPiece));
  L.o_rows = L.o_act + align16((size_t)n_act * sizeof(TickSlot));
  L.o_start = L.o_rows + align16((size_t)B * 8);
  L.o_plan = L.o_start + align16((size_t)B * 8);
  L.o_states = L.o_plan + align16((size_t)B * stride * 4);
  L.o_off = L.o_states + align16((size_t)n_act * 8);
  L.o_trials = L.o_off + align16((size_t)(h->slots + 1) * 4);
  L.mixed = !tp.rs_rows.empty();
  const int n16 = (int)tp.rows16.size(), n_items = (int)tp.items.size(), n_rs = (int)tp.rs_rows.size();
  L.o_rows16 = L.o_trials + align16((size_t)n_act * 24);
  L.o_start16 = L.o_rows16 + align16((size_t)n16 * 8);
  L.o_items = L.o_start16 + align16((size_t)n16 * 8);
  L.o_rs = L.o_items + align16((size_t)n_items * sizeof(RsFrames));
  L.bytes = L.mixed ? L.o_rs + (size_t)n_rs * sizeof(RsRow) : L.o_trials + (size_t)n_act * 24;
  if (gt) {
    L.o_groups = align16(L.bytes);
    L.o_segs = L.o_groups + align16(gt->groups.size() * sizeof(GalGroup));
    L.o_work = L.o_segs + align16(gt->segs.size() * 8);
    L.bytes = L.o_work + gt->work.size() * sizeof(GalWork);
  }
  if (h->in.ensure(L.bytes) || h->wav.ensure((size_t)B * S * 4)) return DG_ECUDA;
  if (L.bytes > h->stage.bytes) {
    PinnedBuf bigger;
    if (bigger.ensure(L.bytes)) return DG_ECUDA;
    if (h->book.n_staged) memcpy(bigger.h, h->stage.h, (size_t)h->book.n_staged * 4);
    h->stage = std::move(bigger);
  }
  unsigned char* pin = h->stage.as<unsigned char>();
  if (np) memcpy(pin + L.o_pieces, h->book.pieces.data(), (size_t)np * sizeof(RingPiece));
  memcpy(pin + L.o_act, act.data(), (size_t)n_act * sizeof(TickSlot));
  memcpy(pin + L.o_rows, tp.rows.data(), (size_t)B * 8);
  memcpy(pin + L.o_start, tp.start.data(), (size_t)B * 8);
  int2* states = reinterpret_cast<int2*>(pin + L.o_states);
  int32_t* off = reinterpret_cast<int32_t*>(pin + L.o_off);
  double* trials = reinterpret_cast<double*>(pin + L.o_trials);
  for (int a = 0, s = 0; a < n_act; a++) {
    const TickSlot& ts = act[a];
    for (; s <= ts.slot; s++) off[s] = ts.row0;
    states[a] = make_int2(ts.slot, a);
    memcpy(trials + 3 * (size_t)a, h->streams[ts.slot].par, 24);
  }
  if (L.mixed) {
    if (n16) memcpy(pin + L.o_rows16, tp.rows16.data(), (size_t)n16 * 8);
    if (n16) memcpy(pin + L.o_start16, tp.start16.data(), (size_t)n16 * 8);
    if (n_items) memcpy(pin + L.o_items, tp.items.data(), (size_t)n_items * sizeof(RsFrames));
    memcpy(pin + L.o_rs, tp.rs_rows.data(), (size_t)n_rs * sizeof(RsRow));
  }
  for (int s = act.back().slot + 1; s <= h->slots; s++) off[s] = B;
  memcpy(pin + L.o_plan, plan_host, (size_t)B * stride * 4);
  if (gt) {
    memcpy(pin + L.o_groups, gt->groups.data(), gt->groups.size() * sizeof(GalGroup));
    memcpy(pin + L.o_segs, gt->segs.data(), gt->segs.size() * 8);
    memcpy(pin + L.o_work, gt->work.data(), gt->work.size() * sizeof(GalWork));
  }
  unsigned char* din = h->in.as<unsigned char>();
  DG_CUDA(cudaEventRecord(h->t_begin, st));
  DG_CUDA(cudaMemcpyAsync(din, pin, L.bytes, cudaMemcpyHostToDevice, st));
  const TickSlot* d_act = reinterpret_cast<const TickSlot*>(din + L.o_act);
  const int2* d_rows = reinterpret_cast<const int2*>(din + L.o_rows);
  int rc;
  // audio in: the staged samples to their rings, then the batch [B, S], windows grouped by slot
  if ((rc = launch_ring_scatter(reinterpret_cast<const float*>(din), reinterpret_cast<const RingPiece*>(din + L.o_pieces), np,
                                h->book.C, h->rings.as<float>(), st)))
    return rc;
  if (!L.mixed) {
    if ((rc = launch_ring_gather(h->rings.as<float>(), h->book.C, d_act, d_rows, reinterpret_cast<const long long*>(din + L.o_start),
                                 S, B, h->wav.as<float>(), st)))
      return rc;
  } else {
    if (n16 && (rc = launch_ring_gather(h->rings.as<float>(), h->book.C, d_act, reinterpret_cast<const int2*>(din + L.o_rows16),
                                        reinterpret_cast<const long long*>(din + L.o_start16), S, n16, h->wav.as<float>(), st)))
      return rc;
    // per declared rate: the new 16 kHz frames of its streams, then its windows
    for (size_t i = 1; i < h->book.rates.size(); i++) {
      const RateGeom& r = h->book.rates[i];
      const int i0 = tp.item_off[i - 1], i1 = tp.item_off[i], w0 = tp.row_off[i - 1], w1 = tp.row_off[i];
      long long max_count = 0;
      for (int k = i0; k < i1; k++) max_count = std::max<long long>(max_count, tp.items[k].count);
      const float* W = r.rs->taps.as<float>();
      if ((rc = launch_resample_frames(h->rings.as<float>(), h->book.C, reinterpret_cast<const RsFrames*>(din + L.o_items) + i0,
                                       i1 - i0, max_count, W, r.g, h->yrings.as<float>(), h->Y, r.Q, st)) ||
          (rc = launch_resample_gather(h->rings.as<float>(), h->book.C, h->yrings.as<float>(), h->Y, r.Q,
                                       reinterpret_cast<const RsRow*>(din + L.o_rs) + w0, w1 - w0, r.r_lo, r.r_hi, W, r.g, r.S, S,
                                       h->wav.as<float>(), st)))
        return rc;
    }
  }
  DG_CUDA(cudaEventRecord(h->e_start, st));
  return DG_OK;
}

// A diarization tick after the audio in: both networks, clustering with a state per slot, the post-path with each slot's
// history, on h->st.
static int tick_diarize(dg_multi* h, const TickPlan& tp, const TickIn& L, int turn_cap) {
  cudaStream_t st = h->st;
  const int B = tp.B, n_act = (int)tp.act.size(), F = h->F, K = h->K, D = h->D, M = h->M, S = h->S;
  const unsigned char* din = h->in.as<unsigned char>();
  const TickSlot* d_act = reinterpret_cast<const TickSlot*>(din + L.o_act);
  const int2* d_rows = reinterpret_cast<const int2*>(din + L.o_rows);
  int rc;
  // networks: sub-batches of at most 256 windows on alternating scratch lanes (the workspace of a 256-window step); a lane is
  // reused once the sub-batch before on it is past its embeddings
  for (int r0 = 0, j = 0; r0 < B; r0 += 256, j++) {
    const int nb = std::min(256, B - r0), lane = j & 1;
    for (cudaStream_t s : {(cudaStream_t)h->net.s_seg[lane], (cudaStream_t)h->net.s_emb})
      DG_CUDA(cudaStreamWaitEvent(s, h->e_lane_done[lane], 0));
    if ((rc = pipeline_nets(&h->net, h->wav.as<float>() + (size_t)r0 * S, S, {nb, F, K}, h->seg.as<float>() + (size_t)r0 * F * K,
                            h->emb.as<float>() + (size_t)r0 * K * D, h->e_start, lane, 0)))
      return rc;
    DG_CUDA(cudaEventRecord(h->e_lane_done[lane], h->net.s_emb));
  }
  DG_CUDA(cudaStreamWaitEvent(st, h->net.e_emb, 0));
  // clustering: state `slot` over that slot's rows (chunk offsets by slot), cosine, at the thresholds of its entry's row
  const double* trials = reinterpret_cast<const double*>(din + L.o_trials);
  ClusterParams p{};
  p.M = M;
  p.D = D;
  p.metric = 0;
  if ((rc = launch_cluster_sweep(p, trials, n_act, reinterpret_cast<const int2*>(din + L.o_states), n_act,
                                 reinterpret_cast<const int*>(din + L.o_off), h->seg.as<float>(), h->emb.as<float>(), B, F, K,
                                 h->centers.as<double>(), h->active.as<int>(), h->init.as<int>(), h->prep.as<float>(),
                                 h->prep_d.as<double>(), h->maps.as<int32_t>(), st, true)))
    return rc;
  // post-path with each slot's history and tau, then the histories move on
  DG_CUDA(cudaMemsetAsync(h->total.p, 0, 4, st));
  int32_t* header = reinterpret_cast<int32_t*>(h->header.as<unsigned char>() + names_bytes(h));
  if ((rc = launch_post_slots(h->seg.as<float>(), h->maps.as<int32_t>(), h->hist_seg.as<float>(), h->hist_map.as<int32_t>(),
                              d_act, d_rows, h->slots, B, F, K, M, h->nw, reinterpret_cast<const int32_t*>(din + L.o_plan),
                              4 + h->nw, h->hamming.as<double>(), trials, header, h->turns.as<uint32_t>(),
                              turn_cap, h->total.as<unsigned int>(), st)) ||
      (rc = launch_post_slots_history(h->seg.as<float>(), h->maps.as<int32_t>(), h->hist_seg.as<float>(),
                                      h->hist_map.as<int32_t>(), d_act, n_act, h->slots, F, K, h->nw, st)))
    return rc;
  return DG_OK;
}

// Gallery naming after a diarization tick, on h->st: the active, unnamed global speakers of the tick's slots with a gallery
// (at most gt.queries, from the host mirror of the named tables), each against its slot's gallery, in one grouped search;
// the new names go to the front of h->header.
static int tick_gallery(dg_multi* h, const GalTick& gt, const TickIn& L) {
  cudaStream_t st = h->st;
  const int n = (int)gt.segs.size(), n_groups = (int)gt.groups.size(), queries = gt.queries, splits = gt.splits;
  if (h->gal_q.ensure((size_t)queries * 8) || h->gal_seg.ensure((size_t)(n + 1) * 4) || h->gal_gq.ensure((size_t)n_groups * 8) ||
      h->gal_d.ensure((size_t)splits * queries * 8) || h->gal_e.ensure((size_t)splits * queries * 4) ||
      h->gal_list.ensure((size_t)queries * 12))
    return DG_ECUDA;
  const unsigned char* din = h->in.as<unsigned char>();
  const GalGroup* groups = reinterpret_cast<const GalGroup*>(din + L.o_groups);
  const int2* segs = reinterpret_cast<const int2*>(din + L.o_segs);
  int* names = h->header.as<int>();
  int rc;
  if ((rc = launch_gallery_queries(segs, n, groups, n_groups, h->active.as<int>(), h->gal_named.as<uint32_t>(), h->M,
                                   h->gal_q.as<int2>(), h->gal_seg.as<int>(), h->gal_gq.as<int2>(), names, st)) ||
      (rc = launch_gallery_nearest(groups, reinterpret_cast<const GalWork*>(din + L.o_work), (int)gt.work.size(),
                                   h->gal_gq.as<int2>(), (h->D + GAL_KC - 1) / GAL_KC * GAL_KC, h->centers.as<double>(), h->D, h->gal_q.as<int2>(), queries, h->gal_claimed.as<int32_t>(),
                                   h->gal_d.as<double>(), h->gal_e.as<int>(), st)) ||
      (rc = launch_gallery_claim(h->gal_d.as<double>(), h->gal_e.as<int>(), queries, h->gal_q.as<int2>(), h->gal_seg.as<int>(),
                                 segs, n, groups, h->gal_claimed.as<int32_t>(), nullptr, nullptr, h->gal_named.as<uint32_t>(),
                                 h->M, names, h->gal_list.as<int32_t>(), names + 4, st)))
    return rc;
  return DG_OK;
}

// A VAD tick after the audio in: the segmentation network alone, then each slot's speech curve binarised with its history of
// max curves, on h->st.
static int tick_vad(dg_multi* h, const TickPlan& tp, const TickIn& L, int turn_cap) {
  cudaStream_t st = h->st;
  const int B = tp.B, n_act = (int)tp.act.size(), F = h->F, K = h->K, S = h->S;
  const unsigned char* din = h->in.as<unsigned char>();
  const TickSlot* d_act = reinterpret_cast<const TickSlot*>(din + L.o_act);
  int rc;
  // segmentation: sub-batches of at most 256 windows on alternating scratch lanes, each bracketed by the lane's guard (as
  // pipeline_nets brackets it) so that other users of the model handle are ordered against it.  A lane takes its next
  // sub-batch in stream order, once the one before on it has its scores; e_lane_done[lane] marks the lane's last scores.
  for (int r0 = 0, j = 0; r0 < B; r0 += 256, j++) {
    const int nb = std::min(256, B - r0), lane = j & 1;
    cudaStream_t s_seg = h->net.s_seg[lane];
    DG_CUDA(cudaStreamWaitEvent(s_seg, h->e_start, 0));
    LaneUse use(h->net.seg->guard[lane], &h->net, s_seg);
    if ((rc = use.rc) ||
        (rc = seg_forward_lane(h->net.seg, lane, nullptr, h->wav.as<float>() + (size_t)r0 * S, nb, S,
                               h->seg.as<float>() + (size_t)r0 * F * K, s_seg)) ||
        (rc = use.end()))
      return rc;
    DG_CUDA(cudaEventRecord(h->e_lane_done[lane], s_seg));
  }
  for (int lane = 0; lane < 2; lane++) DG_CUDA(cudaStreamWaitEvent(st, h->e_lane_done[lane], 0));
  // speech curves with each slot's history and tau, then the histories move on
  DG_CUDA(cudaMemsetAsync(h->total.p, 0, 4, st));
  if ((rc = launch_vad_slots(h->seg.as<float>(), h->hist_vad.as<float>(), d_act, reinterpret_cast<const int2*>(din + L.o_rows),
                             h->slots, B, F, K, h->nw, reinterpret_cast<const int32_t*>(din + L.o_plan), 4 + h->nw,
                             h->hamming.as<double>(), reinterpret_cast<const double*>(din + L.o_trials),
                             h->header.as<int32_t>(), h->turns.as<uint32_t>(), turn_cap, h->total.as<unsigned int>(), st)) ||
      (rc = launch_vad_slots_history(h->seg.as<float>(), h->hist_vad.as<float>(), d_act, n_act, h->slots, F, K, h->nw, st)))
    return rc;
  return DG_OK;
}

extern "C" int dg_multi_step(dg_multi* h, const int32_t* plan_host, int n_rows, int32_t* counts_host, int32_t* header_host,
                             uint32_t* turns_host, int turn_cap_host, int* n_turns, float* seg_dev, float* emb_dev,
                             int32_t* map_dev) {
  const char* who = "dg_multi_step";
  if (!h || !counts_host || n_rows < 0 || (n_rows > 0 && (!plan_host || !header_host || !turns_host))) {
    set_error(std::string(who) + ": bad arguments");
    return DG_EINVAL;
  }
  if (vad_mode(h) && (emb_dev || map_dev)) {
    set_error(std::string(who) + ": a VAD handle has no embeddings or speaker maps");
    return DG_EINVAL;
  }
  // this tick's slots and rows: every open slot with windows gives up to max_wps, in slot order
  TickPlan tp;
  h->book.plan(h->max_wps, tp);
  std::vector<TickSlot>& act = tp.act;
  const int B = tp.B;
  for (int s = 0; s < h->slots; s++) counts_host[s] = 0;
  for (TickSlot& ts : act) {
    const SlotStream& x = h->streams[ts.slot];
    counts_host[ts.slot] = ts.n;
    ts.cur = x.cur;
    ts.n_hist = x.n_hist;
    ts.nw = x.nw;
  }
  if (n_rows != B) {
    set_error(std::string(who) + ": " + std::to_string(n_rows) + " plan rows given, the tick has " + std::to_string(B) +
              " windows");
    return DG_EINVAL;
  }
  const int stride = 4 + h->nw;
  int rc;
  for (const TickSlot& ts : act)
    for (int i = 0; i < ts.n; i++)
      if ((rc = check_plan_row(who, plan_host + (size_t)(ts.row0 + i) * stride, ts.row0 + i, ts.nw, ts.n_hist + i, h->F)))
        return rc;
  if (n_turns) *n_turns = 0;
  h->names_last.clear();
  if (B == 0) return DG_OK;     // nothing to do: staged samples wait for the next tick
  DG_CUDA(cudaSetDevice(h->device));
  cudaStream_t st = h->st;
  const int F = h->F, K = h->K, D = h->D, M = h->M;
  const TurnOut lay = {names_bytes(h), (size_t)B * 16};
  const int turn_cap = post_turn_cap(B, M, F);
  if (h->seg.ensure((size_t)B * F * K * 4) || h->header.ensure(lay.at + lay.header_bytes) || h->turns.ensure((size_t)turn_cap * 4) ||
      h->pin_out.ensure(lay.end()))
    return DG_ECUDA;
  if (!vad_mode(h) && (h->emb.ensure((size_t)B * K * D * 4) || h->maps.ensure((size_t)B * K * 4) ||
                       h->prep.ensure(cluster_prep_floats(B, K) * 4 + 16) || h->prep_d.ensure(cluster_prep_doubles(B, K) * 8 + 16)))
    return DG_ECUDA;
  // with galleries: the tick's slots grouped by gallery and threshold; the unnamed global speakers of a slot are an upper
  // bound of its queries
  GalTick gt;
  if (h->naming) {
    std::vector<int> slot, key, unnamed, G;
    std::vector<double> thr;
    std::vector<const dg_gallery*> gals;
    std::map<std::pair<const dg_gallery*, double>, int> key_of;   // (gallery, threshold) -> key
    for (const TickSlot& ts : act) {
      const SlotStream& x = h->streams[ts.slot];
      int k = -1;
      if (x.gal) {
        const auto it = key_of.emplace(std::make_pair(x.gal, x.thr), (int)gals.size()).first;
        k = it->second;
        if (k == (int)gals.size()) {
          gals.push_back(x.gal);
          thr.push_back(x.thr);
          G.push_back(x.gal->G);
        }
      }
      slot.push_back(ts.slot);
      key.push_back(k);
      unnamed.push_back(M - __builtin_popcount(x.named));
    }
    gallery_tick_plan(slot.data(), key.data(), unnamed.data(), (int)act.size(), G.data(), thr.data(), gt);
    for (size_t r = 0; r < gt.groups.size(); r++) {
      gt.groups[r].E = gals[gt.keys[r]]->E.as<double>();
      gt.groups[r].En = gals[gt.keys[r]]->En.as<double>();
    }
  }
  const int queries = gt.queries;
  TickIn in;
  if ((rc = tick_audio_in(h, tp, plan_host, queries > 0 ? &gt : nullptr, in)) ||
      (rc = vad_mode(h) ? tick_vad(h, tp, in, turn_cap) : tick_diarize(h, tp, in, turn_cap)) ||
      (queries > 0 && (rc = tick_gallery(h, gt, in))))
    return rc;
  if (seg_dev) DG_CUDA(cudaMemcpyAsync(seg_dev, h->seg.p, (size_t)B * F * K * 4, cudaMemcpyDeviceToDevice, st));
  if (emb_dev) DG_CUDA(cudaMemcpyAsync(emb_dev, h->emb.p, (size_t)B * K * D * 4, cudaMemcpyDeviceToDevice, st));
  if (map_dev) DG_CUDA(cudaMemcpyAsync(map_dev, h->maps.p, (size_t)B * K * 4, cudaMemcpyDeviceToDevice, st));
  unsigned char* po = h->pin_out.as<unsigned char>();
  DG_CUDA(cudaMemcpyAsync(po, h->header.p, lay.at + lay.header_bytes, cudaMemcpyDeviceToHost, st));
  DG_CUDA(cudaMemcpyAsync(po + lay.total(), h->total.p, 4, cudaMemcpyDeviceToHost, st));
  DG_CUDA(cudaMemcpyAsync(po + lay.prefix(), h->turns.p, (size_t)std::min(DG_POST_PREFIX, turn_cap) * 4, cudaMemcpyDeviceToHost,
                          st));
  DG_CUDA(cudaEventRecord(h->t_end, st));
  DG_CUDA(cudaStreamSynchronize(st));
  h->timed = true;
  h->last_B = B;
  // the tick is on the device: staged samples are in the rings, windows consumed, frames computed, histories moved on
  h->book.uploaded();
  h->book.consumed(tp);
  for (const TickSlot& ts : act) {
    SlotStream& x = h->streams[ts.slot];
    x.ticked = true;
    if (h->nw > 1) {
      x.n_hist = std::min(ts.nw - 1, ts.n_hist + ts.n);
      x.cur ^= 1;
    }
  }
  if (queries > 0) {   // the new names: the prefix came with the header, the rest (if any) is copied now
    int count = 0;
    memcpy(&count, po, 4);
    h->names_last.resize((size_t)count * 3);
    const int pre = std::min(count, GAL_NAME_PREFIX);
    memcpy(h->names_last.data(), po + 16, (size_t)pre * 12);
    if (count > pre) {
      DG_CUDA(cudaMemcpyAsync(h->names_last.data() + (size_t)pre * 3, h->gal_list.as<int32_t>() + (size_t)pre * 3,
                              (size_t)(count - pre) * 12, cudaMemcpyDeviceToHost, st));
      DG_CUDA(cudaStreamSynchronize(st));
    }
    for (int i = 0; i < count; i++) h->streams[h->names_last[3 * i]].named |= 1u << h->names_last[3 * i + 1];
  }
  return download_turns(who, po, lay, h->turns.as<uint32_t>(), header_host, turns_host, turn_cap_host, n_turns, st);
}

// the named and claimed tables, on the first gallery the handle receives: every slot with nothing named or claimed
static int gallery_tables(dg_multi* h) {
  if (h->naming) return DG_OK;
  if (h->gal_named.ensure((size_t)h->slots * 4) || h->gal_claimed.ensure((size_t)h->slots * 32 * 4)) return DG_ECUDA;
  const int rc = clear_names(h, 0, h->slots);
  h->naming = rc == DG_OK;
  return rc;
}

// a gallery and threshold `who` may give a stream of h: DG_EINVAL naming what rules them out
static int check_gallery_for(const dg_multi* h, const dg_gallery* g, double threshold, const char* who) {
  if (g->D != h->D || g->device != h->device) {
    set_error(std::string(who) + ": the gallery's entries have dimension " + std::to_string(g->D) + " on device " +
              std::to_string(g->device) + ", the embeddings " + std::to_string(h->D) + " on device " + std::to_string(h->device));
    return DG_EINVAL;
  }
  if (!(std::isfinite(threshold) && threshold > 0.0 && threshold <= 2.0)) {
    set_error(std::string(who) + ": need a finite threshold in (0, 2]");
    return DG_EINVAL;
  }
  return DG_OK;
}

extern "C" int dg_multi_set_gallery(dg_multi* h, dg_gallery* g, double threshold) {
  const char* who = "dg_multi_set_gallery";
  if (!h || !g) {
    set_error(std::string(who) + ": null handle");
    return DG_EINVAL;
  }
  if (vad_mode(h) || h->opened) {
    set_error(std::string(who) + (vad_mode(h) ? ": a VAD handle has no speakers to name"
                                               : ": a gallery is set before any stream is opened"));
    return DG_EINVAL;
  }
  int rc;
  if ((rc = check_gallery_for(h, g, threshold, who))) return rc;
  DG_CUDA(cudaSetDevice(h->device));
  if ((rc = gallery_tables(h))) return rc;
  h->gal = g;
  h->gal_threshold = threshold;
  return DG_OK;
}

extern "C" int dg_multi_set_slot_gallery(dg_multi* h, int slot, dg_gallery* g, double threshold) {
  const char* who = "dg_multi_set_slot_gallery";
  if (!h || !g) {
    set_error(std::string(who) + ": null handle");
    return DG_EINVAL;
  }
  if (vad_mode(h)) {
    set_error(std::string(who) + ": a VAD handle has no speakers to name");
    return DG_EINVAL;
  }
  if (!slot_ok(h, slot) || h->streams[slot].ticked) {
    set_error(std::string(who) + ": slot " + std::to_string(slot) +
              (slot_ok(h, slot) ? " has had a tick: a stream's gallery is set before its first tick" : " is not open"));
    return DG_EINVAL;
  }
  int rc;
  if ((rc = check_gallery_for(h, g, threshold, who))) return rc;
  DG_CUDA(cudaSetDevice(h->device));
  // the stream starts over with nothing named or claimed in its gallery
  if ((rc = gallery_tables(h)) || (rc = clear_names(h, slot, 1))) return rc;
  h->streams[slot].gal = g;
  h->streams[slot].thr = threshold;
  return DG_OK;
}

extern "C" int dg_multi_set_names(dg_multi* h, int slot, uint32_t named, const int32_t* claimed_host) {
  const char* who = "dg_multi_set_names";
  if (!slot_ok(h, slot) || vad_mode(h) || !h->streams[slot].gal || !claimed_host) {
    set_error(std::string(who) + ": need an open slot with a gallery and a non-null table");
    return DG_EINVAL;
  }
  const int M = h->M, G = h->streams[slot].gal->G;
  std::vector<int32_t> row(32, -1);
  for (int g = 0; g < M; g++) {
    const int e = claimed_host[g];
    const bool ok = e == -1 || (e >= 0 && e < G && ((named >> g) & 1) &&
                                std::find(claimed_host, claimed_host + g, e) == claimed_host + g);
    if (!ok) {
      set_error(std::string(who) + ": speaker " + std::to_string(g) + " claims entry " + std::to_string(e) +
                " (an entry of the slot's gallery of " + std::to_string(G) + ", claimed once, by a named speaker)");
      return DG_EINVAL;
    }
    row[g] = e;
  }
  if (M < 32 && (named >> M)) {
    set_error(std::string(who) + ": named speakers beyond max_speakers");
    return DG_EINVAL;
  }
  DG_CUDA(cudaSetDevice(h->device));
  DG_CUDA(cudaMemcpyAsync(h->gal_named.as<uint32_t>() + slot, &named, 4, cudaMemcpyHostToDevice, h->st));
  DG_CUDA(cudaMemcpyAsync(h->gal_claimed.as<int32_t>() + (size_t)slot * 32, row.data(), 32 * 4, cudaMemcpyHostToDevice, h->st));
  h->streams[slot].named = named;
  return DG_OK;
}

extern "C" int dg_multi_last_names(const dg_multi* h, int32_t* out_host, int cap, int* n) {
  if (!h || !n || cap < 0 || (cap > 0 && !out_host)) {
    set_error("dg_multi_last_names: bad arguments");
    return DG_EINVAL;
  }
  const int count = (int)(h->names_last.size() / 3);
  *n = count;
  if (count > cap) {
    set_error("dg_multi_last_names: " + std::to_string(count) + " names, room for " + std::to_string(cap));
    return DG_EINVAL;
  }
  if (count) memcpy(out_host, h->names_last.data(), h->names_last.size() * 4);
  return DG_OK;
}

extern "C" int dg_multi_last_step_ms(const dg_multi* h, float* ms) {
  if (!h || !ms || !h->timed) {
    set_error("dg_multi_last_step_ms: no tick with windows has run");
    return DG_EINVAL;
  }
  DG_CUDA(cudaEventElapsedTime(ms, h->t_begin, h->t_end));
  return DG_OK;
}

// the last tick's window batch [n_rows, chunk] (what the networks read) to wav_dev; synchronous
extern "C" int dg_multi_last_windows(const dg_multi* h, float* wav_dev, int n_rows) {
  if (!h || !wav_dev || !h->timed || n_rows != h->last_B) {
    set_error("dg_multi_last_windows: n_rows must be the window count of the last tick that had windows");
    return DG_EINVAL;
  }
  DG_CUDA(cudaSetDevice(h->device));
  DG_CUDA(cudaMemcpyAsync(wav_dev, h->wav.p, (size_t)n_rows * h->S * 4, cudaMemcpyDeviceToDevice, h->st));
  DG_CUDA(cudaStreamSynchronize(h->st));
  return DG_OK;
}

// ================================================================================ moving streams (export / import)
// A stream's state after its last tick, packed (include/diart_b200.h documents the layout): the fixed XferHead, then the
// audio [rpos, wpos), the computed 16 kHz frames a future window still reads, the n_hist history entries oldest first, and
// for a diarization stream its centroids, active flags and claimed gallery entries.  Every section starts at a multiple of
// 16 bytes; a state's size is a multiple of 16, so packed states follow each other directly.
static const uint32_t XFER_MAGIC = 0x54534744u;          // "DGST"
static const int XFER_VERSION = 1;
static const size_t XFER_STAGING = (size_t)256 << 20;    // packed states per round of one launch and one copy

struct XferHead {
  uint32_t magic, version;
  int32_t kind;                    // 0 diarization, 1 VAD
  int32_t S, hop, F, K, D, M;      // the pipeline's window and step, the networks' frames, local speakers, embedding, speakers
  int32_t rs_o, rs_n, rs_w;        // the source rate's resampling (reduced ratio o / n, half-width w; all 0: the pipeline's)
  int32_t chunk, step;             // window and step at the source rate
  int32_t nw, n_hist;              // buffers aggregated (latency / step), history entries held
  int32_t init[2];                 // clustering: initialised, "cannot update unknown centers"
  uint32_t named;                  // named global speakers (bit g)
  int32_t gallery_G;               // entries of the gallery the stream is named from (0: none)
  int32_t ticked, pad0;
  int64_t wpos, rpos, done;        // absolute source samples pushed / start of the next window, 16 kHz frames computed
  int64_t frame0, n_frames;        // the frames carried: [frame0, frame0 + n_frames)
  double params[3];                // tau, rho, delta
  double threshold;                // gallery threshold
  float gamma, beta;
  int32_t normalize, pad1;
  int64_t bytes;                   // the packed state, head included
};

// byte offsets of a state's sections
struct XferLayout {
  size_t audio, frames, hist, hmap, centers, active, claimed, bytes;
};

static XferLayout xfer_layout(const XferHead& hd) {
  XferLayout L{};
  const bool vad = hd.kind == 1;
  L.audio = align16(sizeof(XferHead));
  L.frames = L.audio + align16((size_t)(hd.wpos - hd.rpos) * 4);
  L.hist = L.frames + align16((size_t)hd.n_frames * hd.rs_n * 4);
  L.hmap = L.hist + align16((size_t)hd.n_hist * hd.F * (vad ? 1 : hd.K) * 4);
  L.centers = L.hmap + (vad ? 0 : align16((size_t)hd.n_hist * hd.K * 4));
  L.active = L.centers + (vad ? 0 : align16((size_t)hd.M * hd.D * 8));
  L.claimed = L.active + (vad ? 0 : 32 * 4);
  L.bytes = L.claimed + (vad ? 0 : 32 * 4);
  return L;
}

// the device arrays a move reads or writes, as 32-bit words (a test hook points them at host memory)
struct XferDev {
  uint32_t *rings = nullptr, *yrings = nullptr, *hist_seg = nullptr, *hist_map = nullptr, *hist_vad = nullptr;
  uint32_t *centers = nullptr, *active = nullptr, *init = nullptr, *named = nullptr, *claimed = nullptr;
  long long C = 0, Y = 0;
};

static XferDev xfer_dev(const dg_multi* h) {
  XferDev d;
  d.rings = h->rings.as<uint32_t>(); d.yrings = h->yrings.as<uint32_t>();
  d.hist_seg = h->hist_seg.as<uint32_t>(); d.hist_map = h->hist_map.as<uint32_t>(); d.hist_vad = h->hist_vad.as<uint32_t>();
  d.centers = h->centers.as<uint32_t>(); d.active = h->active.as<uint32_t>(); d.init = h->init.as<uint32_t>();
  if (h->naming) {
    d.named = h->gal_named.as<uint32_t>();
    d.claimed = h->gal_claimed.as<uint32_t>();
  }
  d.C = h->book.C;
  d.Y = h->Y;
  return d;
}

// The one mapping between a stream's slot (its values x, its audio counters a) and the head of its packed state: to_head
// fills hd from (x, a), else (x, a) from hd.  The gallery is the caller's (x.gal); without one, no threshold travels.  A
// restored stream's history is copy 0 (x.cur as given).
static void xfer_map(XferHead& hd, SlotStream& x, SlotAudio& a, bool to_head) {
  auto map = [to_head](auto& field, auto& value) {
    if (to_head) field = value; else value = field;
  };
  map(hd.nw, x.nw); map(hd.n_hist, x.n_hist);
  map(hd.params[0], x.par[0]); map(hd.params[1], x.par[1]); map(hd.params[2], x.par[2]);
  map(hd.threshold, x.thr); map(hd.ticked, x.ticked); map(hd.named, x.named);
  map(hd.wpos, a.wpos); map(hd.rpos, a.rpos); map(hd.done, a.done);
  if (!x.gal) (to_head ? hd.threshold : x.thr) = 0.0;
}

// the head of open slot s (init words: the device's, filled in by the gather)
static XferHead xfer_head(const dg_multi* h, int s) {
  XferHead hd{};
  const RateGeom& r = h->book.geom(s);
  hd.magic = XFER_MAGIC;
  hd.version = XFER_VERSION;
  hd.kind = vad_mode(h) ? 1 : 0;
  hd.S = h->S; hd.hop = h->hop; hd.F = h->F; hd.K = h->K; hd.D = h->D; hd.M = h->M;
  if (r.resampled()) {
    hd.rs_o = r.g.o; hd.rs_n = r.g.n; hd.rs_w = r.g.w;
  }
  hd.chunk = r.S; hd.step = r.hop;
  SlotStream x = h->streams[s];
  SlotAudio a = h->book.audio[s];
  xfer_map(hd, x, a, true);
  hd.gallery_G = x.gal ? x.gal->G : 0;
  if (r.resampled()) {   // frames computed that a future window still reads
    hd.frame0 = hd.rpos / r.g.o + r.r_lo;
    hd.n_frames = std::max<int64_t>(0, hd.done - hd.frame0);
  }
  hd.gamma = h->net.gamma; hd.beta = h->net.beta; hd.normalize = h->net.normalize_weights;
  hd.bytes = (int64_t)xfer_layout(hd).bytes;
  return hd;
}

// The pieces between slot s (history copy `cur`, history stride nw - 1) and its packed state at `blob`: the first n_ring
// samples of the audio, the frames, the history and (diarization) the clustering and naming tables.  to_blob: export
// (the slot is the source), else import.  An export gathers no named bits (the host mirror has them).
static void xfer_pieces(const XferDev& d, const RateGeom& r, int slots, int nw, int s, int cur, const XferHead& hd,
                        uint32_t* blob, long long n_ring, bool to_blob, std::vector<XferPiece>& out) {
  const XferLayout L = xfer_layout(hd);
  auto add = [&](uint32_t* dev, long long pos, long long mod, size_t off, long long n) {
    if (n <= 0) return;
    uint32_t* b = blob + off / 4;
    out.push_back(to_blob ? XferPiece{dev, b, n, pos, mod, 0, 0} : XferPiece{b, dev, n, 0, 0, pos, mod});
  };
  add(d.rings + (size_t)s * d.C, hd.rpos, d.C, L.audio, n_ring);
  if (hd.n_frames) add(d.yrings + (size_t)s * d.Y, hd.frame0 * r.g.n, r.Q * r.g.n, L.frames, hd.n_frames * r.g.n);
  const size_t h0 = ((size_t)cur * slots + s) * (nw - 1), FK = (size_t)hd.F * hd.K;
  if (hd.kind == 1) {
    add(d.hist_vad + h0 * hd.F, 0, 0, L.hist, (long long)hd.n_hist * hd.F);
    return;
  }
  add(d.hist_seg + h0 * FK, 0, 0, L.hist, (long long)(hd.n_hist * FK));
  add(d.hist_map + h0 * hd.K, 0, 0, L.hmap, (long long)hd.n_hist * hd.K);
  add(d.centers + (size_t)s * hd.M * hd.D * 2, 0, 0, L.centers, 2LL * hd.M * hd.D);
  add(d.active + (size_t)s * 32, 0, 0, L.active, 32);
  add(d.init + (size_t)s * 2, 0, 0, offsetof(XferHead, init), 2);
  if (d.claimed) {
    add(d.claimed + (size_t)s * 32, 0, 0, L.claimed, 32);
    if (!to_blob) add(d.named + s, 0, 0, offsetof(XferHead, named), 1);
  }
}

// The staged pieces of each slot (samples pushed since the last tick, still in the pinned staging), in one pass over them
struct StagedBySlot {
  std::vector<int> off, idx;   // slot s: pieces idx [off[s], off[s + 1]) of book.pieces, in push (= stream) order
  std::vector<long long> n;    // slot s: its staged samples
  explicit StagedBySlot(const SlotBook& b) : off(b.audio.size() + 1, 0), idx(b.pieces.size()), n(b.audio.size(), 0) {
    for (const RingPiece& p : b.pieces) {
      off[p.slot + 1]++;
      n[p.slot] += p.n;
    }
    for (size_t s = 0; s + 1 < off.size(); s++) off[s + 1] += off[s];
    std::vector<int> fill(off.begin(), off.end() - 1);
    for (size_t q = 0; q < b.pieces.size(); q++) idx[fill[b.pieces[q].slot]++] = (int)q;
  }
};

// After the gather of slot s into `out`: its head (keeping the gathered init words), its staged samples, without naming
// tables no claims, and zeros in the gaps that align the sections, so that a state's bytes depend on the stream alone.
static void xfer_finish(const dg_multi* h, int s, const XferHead& head, const float* stage, const StagedBySlot& sb,
                        unsigned char* out) {
  XferHead hd = head;
  const XferLayout L = xfer_layout(hd);
  if (hd.kind == 0) memcpy(hd.init, out + offsetof(XferHead, init), 8);
  memcpy(out, &hd, sizeof(hd));
  for (int q = sb.off[s]; q < sb.off[s + 1]; q++) {
    const RingPiece& p = h->book.pieces[sb.idx[q]];
    memcpy(out + L.audio + (size_t)(p.dst - hd.rpos) * 4, stage + p.src, (size_t)p.n * 4);
  }
  if (hd.kind == 0 && !h->naming) memset(out + L.claimed, 0xff, 32 * 4);
  const size_t vad = hd.kind == 1, FK = (size_t)hd.F * (vad ? 1 : hd.K);
  const size_t used[][2] = {{sizeof(XferHead), L.audio},
                            {L.audio + (size_t)(hd.wpos - hd.rpos) * 4, L.frames},
                            {L.frames + (size_t)hd.n_frames * hd.rs_n * 4, L.hist},
                            {L.hist + (size_t)hd.n_hist * FK * 4, L.hmap},
                            {L.hmap + (vad ? 0 : (size_t)hd.n_hist * hd.K * 4), L.centers},
                            {L.centers + (vad ? 0 : (size_t)hd.M * hd.D * 8), L.active}};
  for (const auto& g : used) memset(out + g[0], 0, g[1] - g[0]);
}

static int xfer_slots_ok(const dg_multi* h, const int32_t* slots, int n, const char* who) {
  if (!h || n < 0 || (n > 0 && !slots)) {
    set_error(std::string(who) + ": bad arguments (a handle, n >= 0 slots)");
    return DG_EINVAL;
  }
  std::vector<char> seen(h->slots, 0);
  for (int a = 0; a < n; a++) {
    const int s = slots[a];
    if (!slot_ok(h, s) || seen[s]) {
      set_error(std::string(who) + ": slot " + std::to_string(s) + " is not open or is listed twice");
      return DG_EINVAL;
    }
    seen[s] = 1;
  }
  return DG_OK;
}

// Checks packed state a (head hd, its bytes at `blob`, at most `avail` of them) against h before anything is written:
// DG_EINVAL naming who, the state and the reason.  On success rid is its declared rate (-1: the pipeline's) and g the gallery
// it is named from (null: none).
static int xfer_check(const dg_multi* h, const XferHead& hd, const unsigned char* blob, size_t avail, int a,
                      dg_gallery* const* gals, int& rid, dg_gallery*& g, const char* who) {
  const std::string at = std::string(who) + ": state " + std::to_string(a);
  auto fail = [&](const std::string& why) {
    set_error(at + " " + why);
    return DG_EINVAL;
  };
  if (hd.magic != XFER_MAGIC) return fail("is not a packed stream state");
  if (hd.version != (uint32_t)XFER_VERSION)
    return fail("has format version " + std::to_string(hd.version) + ", this build reads version " +
                std::to_string(XFER_VERSION));
  const int kind = vad_mode(h) ? 1 : 0;
  if (hd.kind != kind)
    return fail(kind ? "is a diarization stream, the handle serves voice activity detection"
                     : "is a voice activity detection stream, the handle serves diarization");
  if (hd.S != h->S || hd.hop != h->hop || hd.F != h->F || hd.K != h->K || hd.D != h->D || hd.M != h->M)
    return fail("has windows of " + std::to_string(hd.S) + " / " + std::to_string(hd.hop) + " samples, F = " +
                std::to_string(hd.F) + ", K = " + std::to_string(hd.K) + ", D = " + std::to_string(hd.D) + ", M = " +
                std::to_string(hd.M) + "; the handle " + std::to_string(h->S) + " / " + std::to_string(h->hop) + ", " +
                std::to_string(h->F) + ", " + std::to_string(h->K) + ", " + std::to_string(h->D) + ", " + std::to_string(h->M));
  if (!kind && (hd.gamma != h->net.gamma || hd.beta != h->net.beta || hd.normalize != h->net.normalize_weights))
    return fail("was diarized with other gamma, beta or normalize_embedding_weights");
  const long long wlen = hd.wpos - hd.rpos;
  const XferLayout L = xfer_layout(hd);
  if (hd.rpos < 0 || wlen < 0 || hd.n_hist < 0 || hd.n_frames < 0 || hd.rs_n < 0) return fail("is malformed");
  rid = -2;
  for (size_t i = 0; i < h->book.rates.size(); i++) {
    const RateGeom& r = h->book.rates[i];
    const bool same = r.resampled() ? (hd.rs_o == r.g.o && hd.rs_n == r.g.n && hd.rs_w == r.g.w)
                                    : (hd.rs_o == 0 && hd.rs_n == 0 && hd.rs_w == 0);
    if (same && hd.chunk == r.S && hd.step == r.hop) rid = (int)i - 1;
  }
  if (rid == -2)
    return fail("is at a source rate the handle did not declare (resampling " + std::to_string(hd.rs_o) + " / " +
                std::to_string(hd.rs_n) + ", window " + std::to_string(hd.chunk) + " samples)");
  const RateGeom& r = h->book.rates[rid + 1];
  if (hd.nw < 1 || hd.nw > h->nw)
    return fail("aggregates " + std::to_string(hd.nw) + " buffers, the handle at most " + std::to_string(h->nw) +
                " (its max_latency)");
  if (hd.n_hist > hd.nw - 1 || hd.rpos % r.hop) return fail("is malformed (history or window position)");
  if (wlen > r.cap)
    return fail("holds " + std::to_string(wlen) + " samples of audio, more than the ring's capacity of " +
                std::to_string(r.cap));
  if (hd.bytes != (int64_t)L.bytes || (size_t)hd.bytes > avail) return fail("is malformed or cut short");
  if (r.resampled() ? (hd.n_frames > r.Q || (hd.n_frames && (hd.frame0 != hd.rpos / r.g.o + r.r_lo ||
                                                              hd.done != hd.frame0 + hd.n_frames)) || hd.done < 0)
                    : (hd.n_frames || hd.done))
    return fail("is malformed (16 kHz frames)");
  if (hd.init[1]) return fail("holds a clustering state that failed on its source (unknown centers)");
  if (!std::isfinite(hd.params[0]) || !std::isfinite(hd.params[1]) || !std::isfinite(hd.params[2]))
    return fail("has thresholds that are not finite");
  g = nullptr;
  const int32_t* claimed = reinterpret_cast<const int32_t*>(blob + L.claimed);
  if (hd.gallery_G > 0) {
    if (kind) return fail("is a voice activity detection stream with a gallery");
    g = gals && gals[a] ? gals[a] : h->gal;
    if (!g) return fail("was named from a gallery of " + std::to_string(hd.gallery_G) + " entries: give that gallery");
    if (g->G != hd.gallery_G)
      return fail("was named from a gallery of " + std::to_string(hd.gallery_G) + " entries, the one given has " +
                  std::to_string(g->G));
    if (check_gallery_for(h, g, hd.threshold, at.c_str())) return DG_EINVAL;
    if (h->M < 32 && (hd.named >> h->M)) return fail("names speakers beyond max_speakers");
    for (int k = 0; k < h->M; k++) {
      const int e = claimed[k];
      if (!(e == -1 || (e >= 0 && e < g->G && ((hd.named >> k) & 1) && std::find(claimed, claimed + k, e) == claimed + k)))
        return fail("has a claim of entry " + std::to_string(e) + " by speaker " + std::to_string(k) + " that is not valid");
    }
  } else if (hd.gallery_G < 0 || hd.named || (!kind && std::any_of(claimed, claimed + 32, [](int32_t e) { return e != -1; }))) {
    return fail("names speakers without a gallery");
  }
  return DG_OK;
}

// the stream of state hd (checked) opens in free slot t at declared rate rid, named from g: host bookkeeping only
static void xfer_open(dg_multi* h, int t, int rid, XferHead hd, dg_gallery* g) {
  SlotStream x;
  x.gal = g;
  SlotAudio a{rid + 1};
  xfer_map(hd, x, a, false);
  stream_begin(h, t, x, a);
}

// consecutive states [a0, a1) of one round: as many as fit XFER_STAGING, at least one
static int xfer_round(const std::vector<size_t>& bytes, int a0) {
  int a1 = a0;
  size_t sum = 0;
  while (a1 < (int)bytes.size() && (a1 == a0 || sum + bytes[a1] <= XFER_STAGING)) sum += bytes[a1++];
  return a1;
}

// the device staging and pinned buffer of a round: `bytes` of states, then up to n_pieces descriptors
static int xfer_buffers(dg_multi* h, size_t bytes, size_t n_pieces, size_t& o_desc) {
  o_desc = align16(bytes);
  const size_t need = o_desc + n_pieces * sizeof(XferPiece);
  if (h->xfer.ensure(need) || h->xfer_pin.ensure(need)) return DG_ECUDA;
  return DG_OK;
}

extern "C" int dg_multi_export_bytes(const dg_multi* h, const int32_t* slots, int n, int64_t* bytes_out) {
  int rc;
  if ((rc = xfer_slots_ok(h, slots, n, "dg_multi_export_bytes"))) return rc;
  if (n > 0 && !bytes_out) {
    set_error("dg_multi_export_bytes: null output");
    return DG_EINVAL;
  }
  for (int a = 0; a < n; a++) bytes_out[a] = xfer_head(h, slots[a]).bytes;
  return DG_OK;
}

extern "C" int dg_multi_export(dg_multi* h, const int32_t* slots, int n, int close, void* out_host, int64_t out_bytes) {
  const char* who = "dg_multi_export";
  int rc;
  if ((rc = xfer_slots_ok(h, slots, n, who))) return rc;
  std::vector<XferHead> hd(n);
  std::vector<size_t> bytes(n), off(n + 1, 0);
  for (int a = 0; a < n; a++) {
    hd[a] = xfer_head(h, slots[a]);
    bytes[a] = (size_t)hd[a].bytes;
    off[a + 1] = off[a] + bytes[a];
  }
  if (n > 0 && (!out_host || out_bytes < 0 || (size_t)out_bytes < off[n])) {
    set_error(std::string(who) + ": the states take " + std::to_string(off[n]) + " bytes, room for " +
              std::to_string(out_bytes));
    return DG_EINVAL;
  }
  if (n == 0) return DG_OK;
  DG_CUDA(cudaSetDevice(h->device));
  unsigned char* out = static_cast<unsigned char*>(out_host);
  const StagedBySlot sb(h->book);
  for (int a0 = 0, a1; a0 < n; a0 = a1) {
    a1 = xfer_round(bytes, a0);
    const size_t round = off[a1] - off[a0];
    size_t o_desc;
    if ((rc = xfer_buffers(h, round, (size_t)(a1 - a0) * 9, o_desc))) return rc;
    const XferDev d = xfer_dev(h);
    std::vector<XferPiece> pc;
    for (int a = a0; a < a1; a++) {
      const int s = slots[a];
      xfer_pieces(d, h->book.geom(s), h->slots, h->nw, s, h->streams[s].cur, hd[a],
                  h->xfer.as<uint32_t>() + (off[a] - off[a0]) / 4, hd[a].wpos - hd[a].rpos - sb.n[s], true, pc);
    }
    unsigned char* pin = h->xfer_pin.as<unsigned char>();
    memcpy(pin + o_desc, pc.data(), pc.size() * sizeof(XferPiece));
    const XferPiece* d_pc = reinterpret_cast<const XferPiece*>(h->xfer.as<unsigned char>() + o_desc);
    DG_CUDA(cudaMemcpyAsync(const_cast<XferPiece*>(d_pc), pin + o_desc, pc.size() * sizeof(XferPiece), cudaMemcpyHostToDevice,
                            h->st));
    if ((rc = launch_slot_transfer(d_pc, (int)pc.size(), "slot_transfer_export", h->st))) return rc;
    {
      ProfScope _ps("slot_transfer_d2h", h->st);   // the copy, timed when profiling
      DG_CUDA(cudaMemcpyAsync(pin, h->xfer.p, round, cudaMemcpyDeviceToHost, h->st));
    }
    DG_CUDA(cudaStreamSynchronize(h->st));
    memcpy(out + off[a0], pin, round);
    for (int a = a0; a < a1; a++) xfer_finish(h, slots[a], hd[a], h->stage.as<float>(), sb, out + off[a]);
  }
  for (int a = 0; a < n; a++) {
    int init[2];
    memcpy(init, out + off[a] + offsetof(XferHead, init), 8);
    if (init[1]) {   // as dg_multi_get_state reports it; no slot is closed
      set_error(std::string(who) + ": the stream in slot " + std::to_string(slots[a]) + ": Cannot update unknown centers");
      return DG_EINVAL;
    }
  }
  if (close)
    for (int a = 0; a < n; a++) stream_end(h, slots[a]);
  return DG_OK;
}

extern "C" int dg_multi_import(dg_multi* h, const void* blob_host, int64_t blob_bytes, int n, dg_gallery* const* gals,
                               int32_t* slots_out) {
  const char* who = "dg_multi_import";
  if (!h || n < 0 || blob_bytes < 0 || (n > 0 && (!blob_host || !slots_out))) {
    set_error(std::string(who) + ": bad arguments (a handle, n >= 0 packed states and room for their slots)");
    return DG_EINVAL;
  }
  const unsigned char* blob = static_cast<const unsigned char*>(blob_host);
  std::vector<XferHead> hd(n);
  std::vector<size_t> bytes(n), off(n + 1, 0);
  std::vector<int> rid(n), slot(n);
  std::vector<dg_gallery*> gal(n);
  int rc;
  for (int a = 0; a < n; a++) {
    const size_t avail = (size_t)blob_bytes - off[a];
    if (avail < sizeof(XferHead)) {
      set_error(std::string(who) + ": state " + std::to_string(a) + " is cut short");
      return DG_EINVAL;
    }
    memcpy(&hd[a], blob + off[a], sizeof(XferHead));
    if ((rc = xfer_check(h, hd[a], blob + off[a], avail, a, gals, rid[a], gal[a], who))) return rc;
    bytes[a] = (size_t)hd[a].bytes;
    off[a + 1] = off[a] + bytes[a];
  }
  for (int a = 0, s = 0; a < n; a++, s++) {   // the lowest free slots
    while (s < h->slots && h->book.audio[s].open) s++;
    if (s == h->slots) {
      set_error(std::string(who) + ": " + std::to_string(n) + " states, fewer free slots");
      return DG_EINVAL;
    }
    slot[a] = s;
  }
  if (n == 0) return DG_OK;
  DG_CUDA(cudaSetDevice(h->device));
  if (std::any_of(gal.begin(), gal.end(), [](dg_gallery* g) { return g != nullptr; }) && (rc = gallery_tables(h))) return rc;
  for (int a0 = 0, a1; a0 < n; a0 = a1) {
    a1 = xfer_round(bytes, a0);
    const size_t round = off[a1] - off[a0];
    size_t o_desc;
    if ((rc = xfer_buffers(h, round, (size_t)(a1 - a0) * 9, o_desc))) return rc;
    const XferDev d = xfer_dev(h);
    std::vector<XferPiece> pc;
    for (int a = a0; a < a1; a++) {
      const int t = slot[a];
      xfer_pieces(d, h->book.rates[rid[a] + 1], h->slots, h->nw, t, 0, hd[a], h->xfer.as<uint32_t>() + (off[a] - off[a0]) / 4,
                  hd[a].wpos - hd[a].rpos, false, pc);
    }
    unsigned char* pin = h->xfer_pin.as<unsigned char>();
    memcpy(pin, blob + off[a0], round);
    memcpy(pin + o_desc, pc.data(), pc.size() * sizeof(XferPiece));
    const XferPiece* d_pc = reinterpret_cast<const XferPiece*>(h->xfer.as<unsigned char>() + o_desc);
    {
      ProfScope _ps("slot_transfer_h2d", h->st);   // the copy, timed when profiling
      DG_CUDA(cudaMemcpyAsync(h->xfer.p, pin, o_desc + pc.size() * sizeof(XferPiece), cudaMemcpyHostToDevice, h->st));
    }
    if ((rc = launch_slot_transfer(d_pc, (int)pc.size(), "slot_transfer_import", h->st))) return rc;
    DG_CUDA(cudaStreamSynchronize(h->st));   // the pinned buffer is reused by the next round
  }
  // the slots open once every round has landed: an error above leaves them closed (what was written is reset by the next
  // open of those slots, and never read before)
  for (int a = 0; a < n; a++) {
    xfer_open(h, slot[a], rid[a], hd[a], gal[a]);
    slots_out[a] = slot[a];
  }
  return DG_OK;
}

// dg_multi's tick planning on its own (test hook, no GPU): a SlotBook whose pipeline windows are out_chunk / out_step samples,
// with the declared rates [n_rates][5] = {o, n, w, chunk, step}, driven by ops [n_ops][3] = {kind, slot, n}.
extern "C" int dg_selftest_multi_frames_host(int slots, int max_wps, int out_chunk, int out_step, int n_rates, const int32_t* rates,
                                             int n_ops, const int32_t* ops, int32_t* result, int64_t* records, int cap,
                                             int* n_records) {
  const char* who = "dg_selftest_multi_frames_host";
  if (slots < 1 || max_wps < 1 || out_chunk < 1 || out_step < 1 || n_rates < 0 || (n_rates && !rates) || n_ops < 0 ||
      (n_ops && (!ops || !result)) || cap < 0 || (cap && !records) || !n_records) {
    set_error(std::string(who) + ": bad arguments");
    return DG_EINVAL;
  }
  SlotBook book;
  book.init(slots, pipeline_rate(out_chunk, out_step, max_wps));
  for (int i = 0; i < n_rates; i++) {
    const int32_t* q = rates + 5 * i;
    RsGeom g{q[0], q[1], q[2], 2 * q[2] + q[0]};
    RateGeom r;
    if (g.o < 1 || g.n < 1 || g.w < 0) {
      set_error(std::string(who) + ": bad rate geometry");
      return DG_EINVAL;
    }
    int rc;
    if ((rc = rate_geom(g, q[3], q[4], out_chunk, max_wps, r, who))) return rc;
    book.add_rate(r);
  }
  *n_records = 0;
  int tick = 0;
  TickPlan tp;
  auto record = [&](long long kind, long long slot, long long a, long long b) {
    if (*n_records < cap) {
      int64_t* r = records + 5 * (size_t)*n_records;
      r[0] = tick; r[1] = kind; r[2] = slot; r[3] = a; r[4] = b;
    }
    ++*n_records;
  };
  for (int i = 0; i < n_ops; i++) {
    const int kind = ops[3 * i], slot = ops[3 * i + 1], n = ops[3 * i + 2];
    int rc = DG_OK;
    if (kind == 0) {
      if (slot < 0 || slot >= slots || book.audio[slot].open || n < -1 || n + 1 >= (int)book.rates.size()) rc = DG_EINVAL;
      else book.start(slot, SlotAudio{n + 1});
    } else if (kind == 1) {
      if (!book.ok(slot)) rc = DG_EINVAL;
      else book.stop(slot);
    } else if (kind == 2) {
      if (!book.ok(slot) || n < 0 || !book.fits(slot, n)) rc = DG_EINVAL;
      else if (n > 0) book.push(slot, n);
    } else if (kind == 4) {
      book.plan(max_wps, tp);
      for (const RsFrames& it : tp.items) record(0, it.slot, it.first, it.count);
      for (int b = 0; b < tp.B; b++) record(1, tp.act[tp.rows[b].x].slot, tp.start[b], b);
      book.uploaded();
      book.consumed(tp);
      tick++;
    } else {
      rc = DG_EINVAL;
    }
    result[i] = rc;
  }
  if (*n_records > cap) {
    set_error(std::string(who) + ": " + std::to_string(*n_records) + " records, room for " + std::to_string(cap));
    return DG_EINVAL;
  }
  return DG_OK;
}

// The host half of dg_multi's audio path on its own (test hook, no GPU): a SlotBook over `slots` rings of C samples driven by
// ops [n_ops][3] = {kind, slot, n}, with ring_scatter's writes done on the host.
extern "C" int dg_selftest_multi_staging_host(int slots, int C, int n_ops, const int32_t* ops, const float* samples_host,
                                              int32_t* result, float* rings_host) {
  if (slots < 1 || C < 1 || n_ops < 0 || (n_ops && (!ops || !result)) || !rings_host) {
    set_error("dg_selftest_multi_staging_host: bad arguments");
    return DG_EINVAL;
  }
  SlotBook book;
  RateGeom base;
  base.cap = C;
  book.init(slots, base);
  std::vector<float> staged;
  long long next = 0;                         // samples of samples_host used so far
  for (int i = 0; i < n_ops; i++) {
    const int kind = ops[3 * i], slot = ops[3 * i + 1], n = ops[3 * i + 2];
    int rc = DG_OK;
    if (kind == 0) {
      if (slot < 0 || slot >= slots || book.audio[slot].open) rc = DG_EINVAL;
      else book.start(slot);
    } else if (kind == 1) {
      if (!book.ok(slot)) rc = DG_EINVAL;
      else book.stop(slot);
    } else if (kind == 2) {
      if (!book.ok(slot) || n < 0 || !book.fits(slot, n)) {
        rc = DG_EINVAL;
      } else if (n > 0) {
        staged.insert(staged.end(), samples_host + next, samples_host + next + n);
        book.push(slot, n);
      }
      if (n > 0) next += n;                   // a refused block is skipped in the sample stream too
    } else if (kind == 3) {
      if (!book.ok(slot) || n < 0 || book.audio[slot].rpos + n > book.audio[slot].wpos) rc = DG_EINVAL;
      else book.audio[slot].rpos += n;
    } else if (kind == 4) {
      for (const RingPiece& p : book.pieces)   // what ring_scatter_kernel writes
        for (int k = 0; k < p.n; k++) rings_host[(size_t)p.slot * C + (p.dst + k) % C] = staged[p.src + k];
      book.uploaded();
      staged.clear();
    } else {
      rc = DG_EINVAL;
    }
    result[i] = rc;
  }
  return DG_OK;
}

// The grouped gallery search plan of a tick on its own (test hook, no GPU): the tick's slots [n][3] = {slot, gallery key
// (-1: none), unnamed speakers} in slot order, galleries G [n_keys] at thresholds thr [n_keys] -> groups [.][6] = {key, G,
// tiles, per_split, splits, q_ub}, segments [.][2] = {slot, group}, work list [cap][3] = {group, tile, split}, counts [4] =
// {groups, segments, work items, splits}.  groups and segments need room for n entries.
extern "C" int dg_selftest_gallery_plan_host(int n, const int32_t* slots, int n_keys, const int32_t* G, const double* thr,
                                             int32_t* groups_out, int32_t* segs_out, int32_t* work_out, int cap,
                                             int32_t* counts) {
  const char* who = "dg_selftest_gallery_plan_host";
  if (n < 0 || (n && (!slots || !groups_out || !segs_out)) || n_keys < 0 || (n_keys && (!G || !thr)) || cap < 0 ||
      (cap && !work_out) || !counts) {
    set_error(std::string(who) + ": bad arguments");
    return DG_EINVAL;
  }
  std::vector<int> slot(n), key(n), unnamed(n);
  for (int a = 0; a < n; a++) {
    slot[a] = slots[3 * a];
    key[a] = slots[3 * a + 1];
    unnamed[a] = slots[3 * a + 2];
    if (key[a] < -1 || key[a] >= n_keys || unnamed[a] < 0 || unnamed[a] > 32) {
      set_error(std::string(who) + ": slot entry " + std::to_string(a) + " is out of range");
      return DG_EINVAL;
    }
  }
  for (int k = 0; k < n_keys; k++)
    if (G[k] < 1) {
      set_error(std::string(who) + ": gallery " + std::to_string(k) + " is empty");
      return DG_EINVAL;
    }
  GalTick t;
  gallery_tick_plan(slot.data(), key.data(), unnamed.data(), n, G, thr, t);
  counts[0] = (int)t.groups.size();
  counts[1] = (int)t.segs.size();
  counts[2] = (int)t.work.size();
  counts[3] = t.splits;
  for (size_t r = 0; r < t.groups.size(); r++) {
    const GalGroup& g = t.groups[r];
    const int32_t row[6] = {t.keys[r], g.G, g.tiles, g.per_split, g.splits, g.q_ub};
    memcpy(groups_out + 6 * r, row, sizeof(row));
  }
  memcpy(segs_out, t.segs.data(), t.segs.size() * 8);
  if ((int)t.work.size() > cap) {
    set_error(std::string(who) + ": " + std::to_string(t.work.size()) + " work items, room for " + std::to_string(cap));
    return DG_EINVAL;
  }
  memcpy(work_out, t.work.data(), t.work.size() * sizeof(GalWork));
  return DG_OK;
}

// dg_multi_set_slot_gallery and dg_multi_set_names on a handle without a device (test hook): `slots` slots of a diarization
// handle with embeddings of dimension D and M speakers on device 0, galleries gal [n_gal][3] = {G, D, device}, driven by
// ops [n_ops][4] = {kind, slot, arg, x}: 0 open the slot (no default gallery), 1 dg_multi_set_slot_gallery(slot, gallery
// arg (-1: null), threshold x), 2 give the slot gallery arg as dg_multi_set_slot_gallery leaves it (host state only),
// 3 dg_multi_set_names(slot, named = arg, speaker 0 claiming entry x, the others none), 4 the slot has had a tick, 5 close
// the slot.  result [n_ops]: each op's return code; messages [msg_cap]: each op's error message ("" when none), one per line.
// Only refusals reach the device-free end of an entry point: an accepted call 1 or 3 fails with DG_ECUDA where no device is.
extern "C" int dg_selftest_multi_gallery_host(int slots, int D, int M, int n_gal, const int32_t* gal, int n_ops,
                                              const double* ops, int32_t* result, char* messages, int msg_cap) {
  const char* who = "dg_selftest_multi_gallery_host";
  if (slots < 1 || D < 2 || M < 1 || M > 32 || n_gal < 0 || (n_gal && !gal) || n_ops < 0 || (n_ops && (!ops || !result)) ||
      msg_cap < 1 || !messages) {
    set_error(std::string(who) + ": bad arguments");
    return DG_EINVAL;
  }
  std::vector<dg_gallery> gals((size_t)n_gal);
  for (int i = 0; i < n_gal; i++) {
    gals[i].G = gal[3 * i];
    gals[i].D = gal[3 * i + 1];
    gals[i].device = gal[3 * i + 2];
  }
  dg_multi h;
  multi_init(h, 0, slots, 1, 0, 1, 0, 0, 1);   // no audio: the ops never reach it
  h.D = D;
  h.M = M;
  h.net.emb = reinterpret_cast<dg_emb*>(&h);   // a diarization handle (never dereferenced here)
  std::string text;
  for (int i = 0; i < n_ops; i++) {
    const int kind = (int)ops[4 * i], slot = (int)ops[4 * i + 1], arg = (int)ops[4 * i + 2];
    const double x = ops[4 * i + 3];
    const bool in_range = slot >= 0 && slot < slots;
    int rc = DG_OK;
    set_error("");
    if (kind == 0 && in_range && !h.book.audio[slot].open) {
      stream_begin(&h, slot, SlotStream{}, SlotAudio{});
    } else if (kind == 1 && arg >= -1 && arg < n_gal) {
      rc = dg_multi_set_slot_gallery(&h, slot, arg < 0 ? nullptr : &gals[arg], x);
    } else if (kind == 2 && in_range && arg >= 0 && arg < n_gal) {
      h.streams[slot].gal = &gals[arg];
    } else if (kind == 3) {
      std::vector<int32_t> claimed((size_t)M, -1);
      claimed[0] = (int32_t)x;
      rc = dg_multi_set_names(&h, slot, (uint32_t)arg, claimed.data());
    } else if (kind == 4 && in_range) {
      h.streams[slot].ticked = true;
    } else if (kind == 5 && in_range && h.book.audio[slot].open) {
      stream_end(&h, slot);
    } else {
      rc = DG_EINVAL;
      set_error(std::string(who) + ": op " + std::to_string(i) + " is not valid");
    }
    result[i] = rc;
    text += rc ? std::string(dg_last_error()) : std::string();
    text += '\n';
  }
  h.net.emb = nullptr;
  const size_t n = std::min(text.size(), (size_t)msg_cap - 1);
  memcpy(messages, text.data(), n);
  messages[n] = 0;
  return DG_OK;
}

// dg_multi_export / dg_multi_import between two VAD handles without a device (test hook): the pieces run on the host over
// host arrays.  geom [14] = {slots, max_wps, nw, out_chunk, out_step, F, o, n, w, chunk, step, target slots, target max_wps,
// target nw}: a source handle at the pipeline's windows out_chunk / out_step and (o > 0) one declared rate {o, n, w, chunk,
// step}, and a target with its own slots, max_wps and nw.  ops [n_ops][3] = {kind, slot, n} drive the source: 0 open slot at
// rate id n (-1: the pipeline's rate), 1 close, 2 push the next n samples of samples_host, 4 tick.  A tick writes the staged
// samples to the rings, 16 kHz frame R as the values R n + p (p < n), and moves the histories on as post_slots_history
// does, chunk c of a stream being the F values c F + j.  Then slot src_slot is exported, its head patched (patch: 0 none,
// 1 version, 2 kind, 3 window, 4 nw beyond the target's, 5 backlog beyond the target's ring, 6 unknown centers, 7 undeclared
// rate, 8 magic) and imported into the target's slot 0.  info [16] = {import rc, C, Q, Y, wpos, rpos, done, n_hist, frame0,
// n_frames, state bytes, source C, source Q}; the target's ring [C], frame ring [Y] and history copy 0 [(nw - 1) F] go to
// the outputs of `cap` floats each; message: the import's error ("" when none).
extern "C" int dg_selftest_multi_transfer_host(const int32_t* geom, int n_ops, const int32_t* ops, const float* samples_host,
                                               int32_t* result, int src_slot, int patch, float* ring_out, float* yring_out,
                                               float* hist_out, int64_t cap, int64_t* info, char* message, int msg_cap) {
  const char* who = "dg_selftest_multi_transfer_host";
  if (!geom || n_ops < 0 || (n_ops && (!ops || !result || !samples_host)) || !ring_out || !yring_out || !hist_out ||
      cap < 1 || !info || !message || msg_cap < 1) {
    set_error(std::string(who) + ": bad arguments");
    return DG_EINVAL;
  }
  const int F = geom[5];
  // a host-only VAD handle: the bookkeeping of dg_multi_create_vad, host vectors for the device arrays
  struct Side {
    dg_multi h;
    std::vector<float> rings, yrings, hist;
    XferDev d;
  };
  auto make = [&](Side& x, int slots, int max_wps, int nw) -> int {
    dg_multi& h = x.h;
    multi_init(h, 0, slots, max_wps, geom[3], geom[4], F, 1, nw);
    h.M = 1;
    if (geom[6] > 0) {
      RsGeom g{geom[6], geom[7], geom[8], 2 * geom[8] + geom[6]};
      RateGeom r;
      int rc;
      if ((rc = rate_geom(g, geom[9], geom[10], geom[3], max_wps, r, who))) return rc;
      h.book.add_rate(r);
      h.Y = r.Q * r.g.n;
    }
    x.rings.assign((size_t)slots * h.book.C, 0.f);
    x.yrings.assign((size_t)slots * std::max(1LL, h.Y), 0.f);
    x.hist.assign(2 * (size_t)slots * std::max(1, nw - 1) * F, 0.f);
    x.d.rings = reinterpret_cast<uint32_t*>(x.rings.data());
    x.d.yrings = reinterpret_cast<uint32_t*>(x.yrings.data());
    x.d.hist_vad = reinterpret_cast<uint32_t*>(x.hist.data());
    x.d.C = h.book.C;
    x.d.Y = h.Y;
    return DG_OK;
  };
  auto run = [](const std::vector<XferPiece>& pc) {   // what slot_transfer_kernel does
    for (const XferPiece& p : pc)
      for (long long i = 0; i < p.n; i++)
        p.dst[p.dst_mod ? (p.dst_pos + i) % p.dst_mod : p.dst_pos + i] = p.src[p.src_mod ? (p.src_pos + i) % p.src_mod : p.src_pos + i];
  };
  Side src, dst;
  int rc;
  if ((rc = make(src, geom[0], geom[1], geom[2])) || (rc = make(dst, geom[11], geom[12], geom[13]))) return rc;
  dg_multi& h = src.h;   // a VAD handle (no embedding model)
  std::vector<float> staged;
  long long next = 0;
  for (int i = 0; i < n_ops; i++) {
    const int kind = ops[3 * i], slot = ops[3 * i + 1], n = ops[3 * i + 2];
    rc = DG_OK;
    if (kind == 0) {
      if (slot < 0 || slot >= h.slots || h.book.audio[slot].open || n < -1 || n + 1 >= (int)h.book.rates.size()) rc = DG_EINVAL;
      else stream_begin(&h, slot, SlotStream{h.nw, 0, 0, {h.tau, 0.0, 0.0}}, SlotAudio{n + 1});   // as dg_multi_open_rate
    } else if (kind == 1) {
      if (!h.book.ok(slot)) rc = DG_EINVAL;
      else stream_end(&h, slot);
    } else if (kind == 2) {
      if (!h.book.ok(slot) || n < 0 || !h.book.fits(slot, n)) rc = DG_EINVAL;
      else if (n > 0) {
        staged.resize((size_t)h.book.n_staged);
        staged.insert(staged.end(), samples_host + next, samples_host + next + n);
        h.book.push(slot, n);
        next += n;
      }
    } else if (kind == 4) {
      const long long C = h.book.C;
      for (const RingPiece& p : h.book.pieces)
        for (int k = 0; k < p.n; k++) src.rings[(size_t)p.slot * C + (p.dst + k) % C] = staged[p.src + k];
      TickPlan tp;
      h.book.plan(h.max_wps, tp);
      for (const RsFrames& it : tp.items) {
        const RateGeom& r = h.book.geom(it.slot);
        for (long long R = it.first; R < it.first + it.count; R++)
          for (int p = 0; p < r.g.n; p++) src.yrings[(size_t)it.slot * h.Y + (R % r.Q) * r.g.n + p] = (float)(R * r.g.n + p);
      }
      const size_t stride = (size_t)std::max(1, h.nw - 1);
      for (const TickSlot& ts : tp.act) {   // post_slots_history on the host, chunk c = the values c F + j
        const int s = ts.slot;
        SlotStream& x = h.streams[s];
        const int cur = x.cur, nh = x.n_hist, keep = std::min(x.nw - 1, nh + ts.n);
        const long long c0 = h.book.audio[s].rpos / h.book.geom(s).hop;
        for (int e = 0; e < keep; e++) {
          const int v = ts.n - keep + e;
          float* out = &src.hist[(((size_t)(cur ^ 1) * h.slots + s) * stride + e) * F];
          for (int j = 0; j < F; j++)
            out[j] = v >= 0 ? (float)((c0 + v) * F + j) : src.hist[(((size_t)cur * h.slots + s) * stride + nh + v) * F + j];
        }
        if (h.nw > 1) {
          x.n_hist = keep;
          x.cur ^= 1;
        }
      }
      h.book.uploaded();
      h.book.consumed(tp);
      staged.clear();
    } else {
      rc = DG_EINVAL;
    }
    result[i] = rc;
  }
  if (!h.book.ok(src_slot)) {
    set_error(std::string(who) + ": slot " + std::to_string(src_slot) + " is not open");
    return DG_EINVAL;
  }
  staged.resize((size_t)h.book.n_staged);
  XferHead hd = xfer_head(&h, src_slot);
  std::vector<uint32_t> blob((size_t)hd.bytes / 4, 0);
  std::vector<XferPiece> pc;
  xfer_pieces(src.d, h.book.geom(src_slot), h.slots, h.nw, src_slot, h.streams[src_slot].cur, hd, blob.data(),
              hd.wpos - hd.rpos - StagedBySlot(h.book).n[src_slot], true, pc);
  run(pc);
  xfer_finish(&h, src_slot, hd, staged.data(), StagedBySlot(h.book), reinterpret_cast<unsigned char*>(blob.data()));
  XferHead* ph = reinterpret_cast<XferHead*>(blob.data());
  dg_multi& t = dst.h;
  switch (patch) {
    case 1: ph->version += 1; break;
    case 2: ph->kind = 0; break;
    case 3: ph->S += 4; break;
    case 4: ph->nw = t.nw + 1; break;
    case 5: ph->wpos = ph->rpos + t.book.rates[h.book.audio[src_slot].rate].cap + 1; break;
    case 6: ph->init[1] = 1; break;
    case 7: ph->rs_o += 1; break;
    case 8: ph->magic = 0; break;
    default: break;
  }
  int rid = -1;
  dg_gallery* g = nullptr;
  set_error("");
  memset(info, 0, 16 * sizeof(int64_t));
  const int irc = xfer_check(&t, *ph, reinterpret_cast<const unsigned char*>(blob.data()), blob.size() * 4, 0, nullptr, rid, g,
                             "dg_multi_import");
  const std::string msg = irc ? std::string(dg_last_error()) : std::string();
  const size_t m = std::min(msg.size(), (size_t)msg_cap - 1);
  memcpy(message, msg.data(), m);
  message[m] = 0;
  const RateGeom& tr = t.book.rates[h.book.audio[src_slot].rate];
  const RateGeom& sr = h.book.geom(src_slot);
  const int64_t row[13] = {irc, t.book.C, tr.Q, t.Y, hd.wpos, hd.rpos, hd.done, hd.n_hist, hd.frame0, hd.n_frames, hd.bytes,
                           h.book.C, sr.Q};
  memcpy(info, row, sizeof(row));
  if (irc) return DG_OK;
  const size_t need = std::max({(size_t)t.book.C, (size_t)std::max(1LL, t.Y), (size_t)std::max(1, t.nw - 1) * F});
  if ((size_t)cap < need) {
    set_error(std::string(who) + ": outputs of " + std::to_string(cap) + " floats, the target needs " + std::to_string(need));
    return DG_EINVAL;
  }
  pc.clear();
  xfer_pieces(dst.d, t.book.rates[rid + 1], t.slots, t.nw, 0, 0, *ph, blob.data(), ph->wpos - ph->rpos, false, pc);
  run(pc);
  xfer_open(&t, 0, rid, *ph, nullptr);
  memcpy(ring_out, dst.rings.data(), (size_t)t.book.C * 4);
  memcpy(yring_out, dst.yrings.data(), (size_t)std::max(1LL, t.Y) * 4);
  memcpy(hist_out, dst.hist.data(), (size_t)std::max(1, t.nw - 1) * F * 4);
  return DG_OK;
}
