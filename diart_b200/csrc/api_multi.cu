// Many live audio streams on one device (dg_multi_*): the reference's live loop (inference.py: one window per stream every
// step, SpeakerDiarization.__call__ with a batch of one, diarization.py:172-232) for up to `slots` streams at once, batched
// across the streams.  Work happens in ticks: every open stream contributes its complete, unconsumed windows (at most
// max_wps), and those windows run as ONE batch -- one upload, one network pass (in sub-batches on the two scratch lanes),
// one clustering launch with a state per stream, one post-path launch with a history per stream, one download.
#include <string.h>

#include <algorithm>
#include <cmath>
#include <memory>
#include <vector>

#include "host.cuh"

// The host bookkeeping of the streams' audio, no device work: per slot the open flag and the absolute sample counters pushed
// (staged included) / start of the next window; the samples pushed since the last tick are [0, n_staged) of a staging buffer,
// described by `pieces` in push order.  A piece is a run of ONE slot's samples that is contiguous both in the staging buffer
// and in that slot's stream, so a piece is extended only by a push that continues it in both.
struct SlotBook {
  int C = 0;                                  // ring capacity per slot
  std::vector<char> open;
  std::vector<long long> wpos, rpos;
  std::vector<RingPiece> pieces;
  long long n_staged = 0;

  void init(int slots, int capacity) {
    C = capacity;
    open.assign(slots, 0);
    wpos.assign(slots, 0);
    rpos.assign(slots, 0);
  }
  bool ok(int slot) const { return slot >= 0 && slot < (int)open.size() && open[slot]; }
  long long available(int s, int S, int hop) const {    // complete windows, pushed and not consumed
    const long long have = wpos[s] - rpos[s];
    return have < S ? 0 : (have - S) / hop + 1;
  }
  void start(int slot) {
    open[slot] = 1;
    wpos[slot] = rpos[slot] = 0;
  }
  // the stream ends: its staged samples are dropped (they stay in the staging buffer, no piece refers to them)
  void stop(int slot) {
    open[slot] = 0;
    pieces.erase(std::remove_if(pieces.begin(), pieces.end(), [&](const RingPiece& p) { return p.slot == slot; }),
                 pieces.end());
  }
  bool fits(int slot, int n) const { return wpos[slot] + n - rpos[slot] <= C; }
  // books n > 0 samples of `slot` at staging offset n_staged (the caller copies them there)
  void push(int slot, int n) {
    RingPiece* last = pieces.empty() ? nullptr : &pieces.back();
    if (last && last->slot == slot && last->src + last->n == n_staged && last->dst + last->n == wpos[slot])
      last->n += n;
    else
      pieces.push_back(RingPiece{n_staged, wpos[slot], slot, n});
    n_staged += n;
    wpos[slot] += n;
  }
  void uploaded() {
    pieces.clear();
    n_staged = 0;
  }
};

struct dg_multi {
  int device = 0, slots = 0, max_wps = 0;
  int S = 0, hop = 0;                         // samples per window, between windows
  int F = 0, K = 0, D = 0, M = 0, nw = 1;
  double tau = 0.5, rho = 0.3, delta = 1.0;
  NetLanes net;
  SlotBook book;
  PinnedBuf stage;                            // staged samples [0, book.n_staged), then a tick's tables
  std::vector<int> n_hist, cur;               // per slot: post-path history entries, current copy
  DevBuf rings, hamming, in, wav, seg, emb, maps, centers, active, init, prep, prep_d, hist_seg, hist_map, header, turns, total;
  PinnedBuf pin_out;                          // header, turn count and turn prefix of a tick (TurnOut layout at 0)
  Stream st;
  Event e_start, e_lane_done[2];
  Event t_begin, t_end;                       // timing events around the last tick's device work on `st`
  bool timed = false;                         // a tick has run
};

static bool slot_ok(const dg_multi* h, int slot) { return h && h->book.ok(slot); }

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
  DG_CUDA(cudaSetDevice(seg->device));
  std::unique_ptr<dg_multi> h(new dg_multi());
  h->device = seg->device; h->slots = max_streams; h->max_wps = max_windows_per_stream;
  h->S = chunk_samples; h->hop = step_samples;
  // room for the windows of a tick and as much audio again pushed ahead (as dg_stream)
  h->book.init(max_streams, (int)(((long long)chunk_samples + 2LL * max_windows_per_stream * step_samples + 1023) / 1024 * 1024));
  h->F = F; h->K = K; h->D = D; h->M = max_speakers; h->nw = num_windows;
  h->tau = tau; h->rho = rho; h->delta = delta;
  h->net.seg = seg; h->net.emb = emb;
  h->net.gamma = gamma; h->net.beta = beta; h->net.normalize_weights = normalize_weights;
  const size_t n = (size_t)max_streams, hist = (size_t)std::max(1, num_windows - 1);
  h->n_hist.assign(n, 0); h->cur.assign(n, 0);
  if (h->rings.ensure(n * h->book.C * 4) || h->hamming.ensure((size_t)F * 8) || h->centers.ensure(n * max_speakers * D * 8) ||
      h->active.ensure(n * 32 * 4) || h->init.ensure(n * 2 * 4) || h->hist_seg.ensure(2 * n * hist * F * K * 4) ||
      h->hist_map.ensure(2 * n * hist * K * 4) || h->total.ensure(16))
    return DG_ECUDA;
  DG_CUDA(cudaMemcpy(h->hamming.p, hamming_host, (size_t)F * 8, cudaMemcpyHostToDevice));
  if (net_lanes_create(h->net) || h->st.create() || h->e_start.create() || h->e_lane_done[0].create() ||
      h->e_lane_done[1].create() || h->t_begin.create(cudaEventDefault) || h->t_end.create(cudaEventDefault))
    return DG_ECUDA;
  *out = h.release();
  return DG_OK;
}

extern "C" int dg_multi_destroy(dg_multi* h) {
  delete h;
  return DG_OK;
}

// a new stream in `slot`: empty ring, fresh clustering state (the reference's SpeakerDiarization.reset()), no history
extern "C" int dg_multi_open(dg_multi* h, int slot) {
  if (!h || slot < 0 || slot >= h->slots || h->book.open[slot]) {
    set_error("dg_multi_open: slot " + std::to_string(slot) + " is out of range or already open");
    return DG_EINVAL;
  }
  DG_CUDA(cudaSetDevice(h->device));
  const size_t s = (size_t)slot;
  DG_CUDA(cudaMemsetAsync(h->centers.as<double>() + s * h->M * h->D, 0, (size_t)h->M * h->D * 8, h->st));
  DG_CUDA(cudaMemsetAsync(h->active.as<int>() + s * 32, 0, 32 * 4, h->st));
  DG_CUDA(cudaMemsetAsync(h->init.as<int>() + s * 2, 0, 2 * 4, h->st));
  h->book.start(slot);
  h->n_hist[slot] = 0;
  return DG_OK;
}

// the stream in `slot` ends: its staged samples are dropped, the slot can be opened again
extern "C" int dg_multi_close(dg_multi* h, int slot) {
  if (!slot_ok(h, slot)) {
    set_error("dg_multi_close: slot " + std::to_string(slot) + " is not open");
    return DG_EINVAL;
  }
  h->book.stop(slot);
  return DG_OK;
}

extern "C" int dg_multi_available(const dg_multi* h, int slot) {
  if (!slot_ok(h, slot)) {
    set_error("dg_multi_available: slot " + std::to_string(slot) + " is not open");
    return DG_EINVAL;
  }
  return (int)h->book.available(slot, h->S, h->hop);
}

// appends n samples to the stream in `slot`: copied into the pinned staging, uploaded at the next dg_multi_step
extern "C" int dg_multi_push_host(dg_multi* h, int slot, const float* samples, int n) {
  if (!slot_ok(h, slot) || n < 0 || (n > 0 && !samples)) {
    set_error("dg_multi_push_host: bad arguments (an open slot, n >= 0 samples)");
    return DG_EINVAL;
  }
  if (!h->book.fits(slot, n)) {
    set_error("dg_multi_push_host: ring of slot " + std::to_string(slot) + " full (" +
              std::to_string(h->book.wpos[slot] - h->book.rpos[slot]) + " samples buffered, capacity " +
              std::to_string(h->book.C) +
              "): step first");
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

extern "C" int dg_multi_step(dg_multi* h, const int32_t* plan_host, int n_rows, int32_t* counts_host, int32_t* header_host,
                             uint32_t* turns_host, int turn_cap_host, int* n_turns, float* seg_dev, float* emb_dev,
                             int32_t* map_dev) {
  const char* who = "dg_multi_step";
  if (!h || !counts_host || n_rows < 0 || (n_rows > 0 && (!plan_host || !header_host || !turns_host))) {
    set_error(std::string(who) + ": bad arguments");
    return DG_EINVAL;
  }
  // this tick's slots and rows: every open slot with windows gives up to max_wps, in slot order
  std::vector<TickSlot> act;
  int B = 0;
  for (int s = 0; s < h->slots; s++) {
    const int n = h->book.open[s] ? (int)std::min<long long>(h->book.available(s, h->S, h->hop), h->max_wps) : 0;
    counts_host[s] = n;
    if (n) {
      act.push_back(TickSlot{s, B, n, h->cur[s], h->n_hist[s], {0, 0, 0}});
      B += n;
    }
  }
  if (n_rows != B) {
    set_error(std::string(who) + ": " + std::to_string(n_rows) + " plan rows given, the tick has " + std::to_string(B) +
              " windows");
    return DG_EINVAL;
  }
  const int stride = 4 + h->nw;
  // plan rows post.cu accepts: 1 <= nb <= nw buffers, none before the stream's first chunk, 1 <= frames, at most F + 1 output
  // frames (the first chunk's crop of [0, region end))
  for (const TickSlot& ts : act)
    for (int i = 0; i < ts.n; i++) {
      const int32_t* pl = plan_host + (size_t)(ts.row0 + i) * stride;
      const int nb = pl[0], nf = pl[1], nfo = pl[2] > 0 ? pl[2] : nf;
      if (nb < 1 || nb > h->nw || nb - 1 > ts.n_hist + i || nf < 1 || pl[2] < 0 || nfo > h->F + 1) {
        set_error(std::string(who) + ": plan row " + std::to_string(ts.row0 + i) + " is not a plan of its stream (buffers " +
                  std::to_string(nb) + ", frames " + std::to_string(nfo) + ")");
        return DG_EINVAL;
      }
    }
  if (n_turns) *n_turns = 0;
  if (B == 0) return DG_OK;     // nothing to do: staged samples wait for the next tick
  DG_CUDA(cudaSetDevice(h->device));
  cudaStream_t st = h->st;
  const int n_act = (int)act.size(), np = (int)h->book.pieces.size(), F = h->F, K = h->K, D = h->D, M = h->M, S = h->S;
  // host -> device, ONE copy: staged samples, pieces [np], slots [n_act], rows [B] {slot entry, window}, window starts [B],
  // plan [B][stride], cluster states [n_act] {slot, 0}, chunk offsets [slots + 1] by slot, thresholds [3]
  const size_t o_pieces = align16((size_t)h->book.n_staged * 4), o_act = o_pieces + align16((size_t)np * sizeof(RingPiece));
  const size_t o_rows = o_act + align16((size_t)n_act * sizeof(TickSlot)), o_start = o_rows + align16((size_t)B * 8);
  const size_t o_plan = o_start + align16((size_t)B * 8), o_states = o_plan + align16((size_t)B * stride * 4);
  const size_t o_off = o_states + align16((size_t)n_act * 8), o_trials = o_off + align16((size_t)(h->slots + 1) * 4);
  const size_t in_b = o_trials + 24;
  const TurnOut lay = {0, (size_t)B * 16};
  const int turn_cap = B * M * ((F + 2) / 2);   // every second output frame of every speaker starts a turn
  if (h->in.ensure(in_b) || h->wav.ensure((size_t)B * S * 4) || h->seg.ensure((size_t)B * F * K * 4) ||
      h->emb.ensure((size_t)B * K * D * 4) || h->maps.ensure((size_t)B * K * 4) ||
      h->prep.ensure(cluster_prep_floats(B, K) * 4 + 16) || h->prep_d.ensure(cluster_prep_doubles(B, K) * 8 + 16) ||
      h->header.ensure(lay.header_bytes) || h->turns.ensure((size_t)turn_cap * 4) || h->pin_out.ensure(lay.end()))
    return DG_ECUDA;
  if (in_b > h->stage.bytes) {
    PinnedBuf bigger;
    if (bigger.ensure(in_b)) return DG_ECUDA;
    if (h->book.n_staged) memcpy(bigger.h, h->stage.h, (size_t)h->book.n_staged * 4);
    h->stage = std::move(bigger);
  }
  unsigned char* pin = h->stage.as<unsigned char>();
  if (np) memcpy(pin + o_pieces, h->book.pieces.data(), (size_t)np * sizeof(RingPiece));
  memcpy(pin + o_act, act.data(), (size_t)n_act * sizeof(TickSlot));
  int2* rows = reinterpret_cast<int2*>(pin + o_rows);
  long long* start = reinterpret_cast<long long*>(pin + o_start);
  int2* states = reinterpret_cast<int2*>(pin + o_states);
  int32_t* off = reinterpret_cast<int32_t*>(pin + o_off);
  for (int a = 0, s = 0; a < n_act; a++) {
    const TickSlot& ts = act[a];
    for (; s <= ts.slot; s++) off[s] = ts.row0;
    for (int i = 0; i < ts.n; i++) {
      rows[ts.row0 + i] = make_int2(a, i);
      start[ts.row0 + i] = h->book.rpos[ts.slot] + (long long)i * h->hop;
    }
    states[a] = make_int2(ts.slot, 0);
  }
  for (int s = act.back().slot + 1; s <= h->slots; s++) off[s] = B;
  memcpy(pin + o_plan, plan_host, (size_t)B * stride * 4);
  const double trials[3] = {h->tau, h->rho, h->delta};
  memcpy(pin + o_trials, trials, 24);
  unsigned char* din = h->in.as<unsigned char>();
  DG_CUDA(cudaEventRecord(h->t_begin, st));
  DG_CUDA(cudaMemcpyAsync(din, pin, in_b, cudaMemcpyHostToDevice, st));
  const TickSlot* d_act = reinterpret_cast<const TickSlot*>(din + o_act);
  const int2* d_rows = reinterpret_cast<const int2*>(din + o_rows);
  int rc;
  // audio in: the staged samples to their rings, then the batch [B, S], windows grouped by slot
  if ((rc = launch_ring_scatter(reinterpret_cast<const float*>(din), reinterpret_cast<const RingPiece*>(din + o_pieces), np,
                                h->book.C, h->rings.as<float>(), st)) ||
      (rc = launch_ring_gather(h->rings.as<float>(), h->book.C, d_act, d_rows, reinterpret_cast<const long long*>(din + o_start), S,
                               B, h->wav.as<float>(), st)))
    return rc;
  DG_CUDA(cudaEventRecord(h->e_start, st));
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
  // clustering: state `slot` over that slot's rows (chunk offsets by slot), cosine
  ClusterParams p{};
  p.M = M;
  p.D = D;
  p.metric = 0;
  if ((rc = launch_cluster_sweep(p, reinterpret_cast<const double*>(din + o_trials), 1,
                                 reinterpret_cast<const int2*>(din + o_states), n_act, reinterpret_cast<const int*>(din + o_off),
                                 h->seg.as<float>(), h->emb.as<float>(), B, F, K, h->centers.as<double>(), h->active.as<int>(),
                                 h->init.as<int>(), h->prep.as<float>(), h->prep_d.as<double>(), h->maps.as<int32_t>(), st)))
    return rc;
  // post-path with each slot's history, then the histories move on
  DG_CUDA(cudaMemsetAsync(h->total.p, 0, 4, st));
  if ((rc = launch_post_slots(h->seg.as<float>(), h->maps.as<int32_t>(), h->hist_seg.as<float>(), h->hist_map.as<int32_t>(),
                              d_act, d_rows, h->slots, B, F, K, M, h->nw, reinterpret_cast<const int32_t*>(din + o_plan),
                              stride, h->hamming.as<double>(), h->tau, h->header.as<int32_t>(), h->turns.as<uint32_t>(),
                              turn_cap, h->total.as<unsigned int>(), st)) ||
      (rc = launch_post_slots_history(h->seg.as<float>(), h->maps.as<int32_t>(), h->hist_seg.as<float>(),
                                      h->hist_map.as<int32_t>(), d_act, n_act, h->slots, F, K, h->nw, st)))
    return rc;
  if (seg_dev) DG_CUDA(cudaMemcpyAsync(seg_dev, h->seg.p, (size_t)B * F * K * 4, cudaMemcpyDeviceToDevice, st));
  if (emb_dev) DG_CUDA(cudaMemcpyAsync(emb_dev, h->emb.p, (size_t)B * K * D * 4, cudaMemcpyDeviceToDevice, st));
  if (map_dev) DG_CUDA(cudaMemcpyAsync(map_dev, h->maps.p, (size_t)B * K * 4, cudaMemcpyDeviceToDevice, st));
  unsigned char* po = h->pin_out.as<unsigned char>();
  DG_CUDA(cudaMemcpyAsync(po + lay.at, h->header.p, lay.header_bytes, cudaMemcpyDeviceToHost, st));
  DG_CUDA(cudaMemcpyAsync(po + lay.total(), h->total.p, 4, cudaMemcpyDeviceToHost, st));
  DG_CUDA(cudaMemcpyAsync(po + lay.prefix(), h->turns.p, (size_t)std::min(DG_POST_PREFIX, turn_cap) * 4, cudaMemcpyDeviceToHost,
                          st));
  DG_CUDA(cudaEventRecord(h->t_end, st));
  DG_CUDA(cudaStreamSynchronize(st));
  h->timed = true;
  // the tick is on the device: staged samples are in the rings, windows consumed, histories moved on
  h->book.uploaded();
  for (const TickSlot& ts : act) {
    h->book.rpos[ts.slot] += (long long)ts.n * h->hop;
    if (h->nw > 1) {
      h->n_hist[ts.slot] = std::min(h->nw - 1, ts.n_hist + ts.n);
      h->cur[ts.slot] ^= 1;
    }
  }
  return download_turns(who, po, lay, h->turns.as<uint32_t>(), header_host, turns_host, turn_cap_host, n_turns, st);
}

extern "C" int dg_multi_last_step_ms(const dg_multi* h, float* ms) {
  if (!h || !ms || !h->timed) {
    set_error("dg_multi_last_step_ms: no tick with windows has run");
    return DG_EINVAL;
  }
  DG_CUDA(cudaEventElapsedTime(ms, h->t_begin, h->t_end));
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
  book.init(slots, C);
  std::vector<float> staged;
  long long next = 0;                         // samples of samples_host used so far
  for (int i = 0; i < n_ops; i++) {
    const int kind = ops[3 * i], slot = ops[3 * i + 1], n = ops[3 * i + 2];
    int rc = DG_OK;
    if (kind == 0) {
      if (slot < 0 || slot >= slots || book.open[slot]) rc = DG_EINVAL;
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
      if (!book.ok(slot) || n < 0 || book.rpos[slot] + n > book.wpos[slot]) rc = DG_EINVAL;
      else book.rpos[slot] += n;
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
