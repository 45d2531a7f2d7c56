// The host layer's shared part: what more than one of the api*.cu translation units needs -- the owning types, the handle
// structs that another file reads, and the functions called across files.  Everything else is local to its file.
#pragma once
#include <deque>
#include <map>
#include <memory>
#include <string>
#include <utility>
#include <vector>

#include "../../include/diart_b200.h"
#include "dg_common.cuh"

namespace dg {

// ------------------------------------------------------------------------------ small utilities
struct DevBuf {
  void* p = nullptr;
  size_t bytes = 0;
  int ensure(size_t n) {
    if (n <= bytes) return 0;
    if (p) cudaFree(p);
    p = nullptr;
    bytes = 0;
    // (re)allocation is rare (first step at a given batch size).  The handles drive several non-blocking
    // streams, which do not order against the legacy stream this memset runs on: drain the device on both sides.
    DG_CUDA(cudaDeviceSynchronize());
    DG_CUDA(cudaMalloc(&p, n));
    DG_CUDA(cudaMemset(p, 0, n));
    DG_CUDA(cudaDeviceSynchronize());
    bytes = n;
    return 0;
  }
  template <class T>
  T* as() const { return reinterpret_cast<T*>(p); }
  ~DevBuf() {
    if (p) cudaFree(p);
  }
};

// An owned CUDA handle, freed by `Free`; movable, not copyable.  A handle struct that holds its streams, events and pinned
// memory this way frees everything it created, also when its creation fails halfway.
template <class H, cudaError_t (*Free)(H)>
struct Owned {
  H h = nullptr;
  Owned() = default;
  Owned(Owned&& o) noexcept : h(o.h) { o.h = nullptr; }
  Owned& operator=(Owned&& o) noexcept {
    std::swap(h, o.h);
    return *this;
  }
  ~Owned() {
    if (h) Free(h);
  }
  operator H() const { return h; }
};
struct Stream : Owned<cudaStream_t, cudaStreamDestroy> {
  int create(int priority = 0) {   // 0: the default priority
    DG_CUDA(cudaStreamCreateWithPriority(&h, cudaStreamNonBlocking, priority));
    return 0;
  }
};
struct Event : Owned<cudaEvent_t, cudaEventDestroy> {
  int create(unsigned flags = cudaEventDisableTiming) {
    DG_CUDA(cudaEventCreateWithFlags(&h, flags));
    return 0;
  }
};
struct PinnedBuf : Owned<void*, cudaFreeHost> {
  size_t bytes = 0;
  int ensure(size_t n) {   // like DevBuf::ensure, without clearing
    if (n <= bytes) return 0;
    if (h) cudaFreeHost(h);
    h = nullptr;
    bytes = 0;
    DG_CUDA(cudaHostAlloc(&h, n, cudaHostAllocDefault));
    bytes = n;
    return 0;
  }
  template <class T>
  T* as() const { return reinterpret_cast<T*>(h); }
};

// A model handle owns ONE set of activation buffers per scratch lane.  A new user of a lane -- another pipeline built on the same
// handle, or a block-level call on another stream -- first waits, stream-ordered, for the previous user's last kernel; without it
// two users in flight would silently overwrite each other's activations.  (Host threads: a handle is single-threaded.)
struct UseGuard {
  Event e;                       // recorded at the end of the last use
  const void* owner = nullptr;   // who made it
};
// One use of a lane by `owner` on `st`: the constructor makes `st` wait for a previous user's end (`rc` = its result); end(), or
// the destructor on any other exit, records this use's end, so that the next user also waits for what an error left enqueued.
struct LaneUse {
  UseGuard& u;
  const void* owner;
  cudaStream_t st;
  int rc;
  bool open = true;
  LaneUse(UseGuard& u_, const void* owner_, cudaStream_t st_) : u(u_), owner(owner_), st(st_), rc(begin()) {}
  ~LaneUse() { end(); }
  int end() {
    if (!open) return 0;
    open = false;
    if (!u.e && u.e.create()) return DG_ECUDA;
    DG_CUDA(cudaEventRecord(u.e, st));
    u.owner = owner;
    return 0;
  }
  int begin() {
    if (u.e && u.owner != owner) DG_CUDA(cudaStreamWaitEvent(st, u.e, 0));
    return 0;
  }
};

struct Tensors {
  std::map<std::string, std::pair<const float*, int64_t>> m;
  Tensors(const dg_tensor* t, int n) {
    for (int i = 0; i < n; i++)
      if (t[i].name) m[t[i].name] = {t[i].data, t[i].numel};
  }
  const float* get(const std::string& name, int64_t numel) const {
    auto it = m.find(name);
    if (it == m.end()) {
      set_error("missing tensor '" + name + "' in state dict");
      return nullptr;
    }
    if (it->second.second != numel || !it->second.first) {
      set_error("tensor '" + name + "' has " + std::to_string(it->second.second) + " elements, expected " +
                std::to_string(numel));
      return nullptr;
    }
    return it->second.first;
  }
  int64_t numel(const std::string& name) const {
    auto it = m.find(name);
    return it == m.end() ? -1 : it->second.second;
  }
};

// The B operand of a tensor-core GEMM: fp16 hi/lo planes [Npad][K] of float32 weights that were multiplied by `scale` (a power
// of two) before the split.  Npad, the row count the GEMM's tiles read, is decided here once, at upload.
struct WeightPlanes {
  DevBuf hi, lo;
  float scale = 1.f;
  int Npad = 0, K = 0;
};

// api.cu
int upload_u16(DevBuf& b, const std::vector<uint16_t>& h);
int upload_split(WeightPlanes& w, const std::vector<float>& w_nk, int N, int Npad, int K);
int set_weights(TcGemm& t, const WeightPlanes& w);
int upload(DevBuf& b, const std::vector<float>& h);

// ------------------------------------------------------------------------------ SincNet front end (api_seg.cu)
struct SincWeights {
  float wn_gamma = 1.f, wn_beta = 0.f;
  DevBuf g0, b0, bias1, g1, b1, bias2, g2, b2;
  WeightPlanes w1, w2;                 // conv weights [64][5*80] and [64][5*64] (tap-major K)
  DevBuf filt_planes;                  // sinc filter bank as fp16 planes [2][80][256] (hi, lo)
  DevBuf cf;                           // folded wav-norm affine: beta * sum_k h[f][k]
  DevBuf hsum;                         // sum_k h[f][k] (stream form of the sinc layer)
};

// waveform statistics and the standardised-waveform planes of a batch; both networks' SincNets read the same
// ones, so the fused pipeline computes them once per step
struct SincPrep {
  DevBuf wmean, wrstd, wh, wl;
  // stream form (needs a hop hint): planes of the raw stream and the device flag "this batch is a run of overlapping
  // windows"; `hop` > 0 means the stream-form launches were enqueued for this batch
  DevBuf swh, swl, flag, spart;
  int hop = 0;
  int ensure(int B, const Geom& g) {
    const size_t bytes = 4 * sinc_tc_plane_elems(B, g) * 2;
    return (wmean.ensure(B * 4) || wrstd.ensure(B * 4) || wh.ensure(bytes) || wl.ensure(bytes)) ? DG_ECUDA : 0;
  }
  int ensure_stream(int B, const Geom& g, int hop_) {
    const size_t bytes = 4 * sinc_stream_geom(B, g, hop_).plane * 2;
    return (swh.ensure(bytes) || swl.ensure(bytes) || flag.ensure(16)) ? DG_ECUDA : 0;
  }
};
struct SincWork {
  DevBuf p0, sc0, sh0, p1, sc1, sh1, p2, sc2, sh2;
  DevBuf a0h, a0l, c1, a1h, a1l, c2;   // fp16 planes of the conv inputs; un-pooled conv outputs of the un-fused path
  DevBuf craw, part;                   // stream form: raw convolution of the stream [P][80], statistics partials
  DevBuf part3;                        // per-tile InstanceNorm partial sums of the pooling GEMM epilogues (conv1, conv2)
  SincPrep own_prep;                   // statistics + waveform planes when no shared ones are supplied
  const float* out = nullptr;          // conv2 output that the next layer normalises on load ...
  int out_pool = 0;                    // ... 1: still un-pooled (rows = 3x), MaxPool1d(3) is applied on load
  int ensure(int B, const Geom& g) {
    const size_t tail = 64;  // spare rows so shifted windows of the last tile stay in bounds
    if (p0.ensure(((size_t)B * g.S0 + tail) * 80 * 4) || sc0.ensure((size_t)B * 80 * 4) || sh0.ensure((size_t)B * 80 * 4) ||
        p1.ensure(((size_t)B * g.S1 + tail) * 64 * 4) || sc1.ensure((size_t)B * 64 * 4) ||
        sh1.ensure((size_t)B * 64 * 4) || p2.ensure(((size_t)B * g.S2 + tail) * 64 * 4) ||
        sc2.ensure((size_t)B * 64 * 4) || sh2.ensure((size_t)B * 64 * 4) ||
        a0h.ensure(((size_t)B * g.S0 + tail) * 128 * 2) || a0l.ensure(((size_t)B * g.S0 + tail) * 128 * 2) ||
        c1.ensure(((size_t)B * g.S0 + tail) * 64 * 4) || a1h.ensure(((size_t)B * g.S1 + tail) * 64 * 2) ||
        a1l.ensure(((size_t)B * g.S1 + tail) * 64 * 2) || c2.ensure(((size_t)B * g.S1 + tail) * 64 * 4))
      return DG_ECUDA;
    return 0;
  }
};

int prep_sincnet(const Tensors& t, const std::string& pre, SincWeights& w);
int run_sinc_prep(SincPrep& p, const float* wav, int B, const Geom& g, cudaStream_t st, int hop = 0,
                  bool overlap_known = false);
int run_sincnet(const SincWeights& w, SincWork& k, const float* wav, int B, const Geom& g, cudaStream_t st,
                const SincPrep* shared = nullptr);

// ---- test hooks dg_seg_debug_stage / dg_emb_debug_stage (api_seg.cu): copy-out of what a forward left on the device
// un-padded rows and real channels of an [B * item_rows][ld] map -> out [B][T][C] float32 on the host; `lo` non-null: fp16
// hi / lo planes, returned as hi + lo (exact in float32); `lo` null: `hi` is a float32 map.  dims = {B, T, C}.
int debug_copy_map(const char* who, const void* hi, const void* lo, int B, int item_rows, int ld, int T, int C, float* out_host,
                   int64_t cap, int* dims);
// stages 0..3 of both hooks, after a forward through `k` (`prep`: the shared statistics, or null for k.own_prep): operand of
// conv1, operand of conv2, operand of the LSTM / TDNN1 (`xh`, `xl`), waveform statistics [2][B] (mean, rstd)
int debug_copy_front(const char* who, int stage, const SincWork& k, const SincPrep* prep, const void* xh, const void* xl, int B,
                     const Geom& g, float* out_host, int64_t cap, int* dims);
// dims[3] of both hooks, bit 0 and 1: the stream form of the sinc layer did the work (hint accepted AND the device flag set);
// conv1 / conv2 ran with MaxPool1d(3) in the GEMM epilogue
int debug_front_paths(const SincPrep* prep, const Geom& g, int* paths);
enum { DG_DBG_STREAM_FORM = 1, DG_DBG_POOL3_FUSED = 2, DG_DBG_LSTM_16ROWS = 4, DG_DBG_STATS_POOL_FUSED = 8 };

// Sets g_sm_limit for its lifetime (0: no cap).
struct SmLimit {
  const int prev;
  explicit SmLimit(int limit) : prev(g_sm_limit) { g_sm_limit = limit; }
  ~SmLimit() { g_sm_limit = prev; }
};

}  // namespace dg

using namespace dg;

// ================================================================================== segmentation (api_seg.cu)
struct dg_seg {
  int device = 0, K = 3;           // K = classifier outputs (local speakers; powerset classes for powerset models)
  int ps_speakers = 0;             // > 0: powerset model with this many local speakers (dg_seg_set_powerset)
  DevBuf ps_masks;                 // speaker bit set of every powerset class
  SincWeights sw;
  DevBuf bih[4];                   // input projection bias b_ih + b_hh [1024]
  WeightPlanes wih[4];             // input projections [1024][in_pad]
  WeightPlanes whh[4];             // W_hh [2][512][128] as lstm_tc_pack_whh lays it out (hi, lo, scale; no GEMM shape)
  DevBuf l1b, l2b, cw, cb;
  WeightPlanes l1, l2;             // head Linears [128][in]
  DevBuf ones128, zeros128;
  // activations: two independent sets ("lanes") so that the fused pipeline can run the segmentation chains of
  // two consecutive steps concurrently (the recurrence occupies only 32 SMs)
  struct Scratch {
    SincWork work;
    DevBuf gx, y2;
    DevBuf xh, xl;                 // fp16 hi/lo planes of the current in-projection input
    DevBuf y1h, y1l;               // fp16 planes of the first head Linear's output
  } scr[2];
  UseGuard guard[2];               // per scratch lane
};

// the forward on scratch lane `lane`, without the use bracket; `prep`: waveform statistics + planes the caller computed (or null)
// `stop_after` (test hook dg_seg_debug_stage): -1 returns before the LSTM, L < 3 after LSTM layer L
int seg_forward_lane(dg_seg* h, int lane, const SincPrep* prep, const float* wav, int B, int S, float* seg, cudaStream_t st,
                     int stop_after = 99);

// ===================================================================================== embedding (api_emb.cu)
struct dg_emb {
  int device = 0, pool_mode = 31, D = 512;
  SincWeights sw;
  DevBuf tb[5], bns[5], bnh[5];
  WeightPlanes tw[5];                    // TDNN weights [Npad][K]
  WeightPlanes ew;                       // Linear(3000, D) weights [Dpad][3008] (WeSpeaker: Linear(5120, D))
  DevBuf ph, pl;                         // pooled statistics planes
  DevBuf xh, xl, aH, aL, bH, bL;         // fp16 hi/lo activation planes
  DevBuf eb;
  SincWork work;
  UseGuard guard;
  DevBuf t5, pooled, eraw;
  DevBuf idx0, idx1, lam1;
  int tab_F = -1, tab_T = -1;
  DevBuf flags, uniq, grp, gathered;   // compatibility path
  // what the pooling reads after a trunk pass: x(item, t, c) = pool_x[item * pool_item_pitch + t * pool_row_pitch + c], c < pool_C
  const float* pool_x = nullptr;
  long long pool_item_pitch = 0;
  int pool_row_pitch = 0, pool_C = 1500;
  const void *t4h = nullptr, *t4l = nullptr;   // operand planes of TDNN5 after a trunk pass that stopped before it
  DevBuf pool_rw, pool_vs, pool_part;           // fused TDNN5 + pooling: row weights, weight sums, per-tile partial sums
  int variant = 0;                     // 0: XVectorSincNet (pyannote/embedding), 1: WeSpeaker ResNet34 (variant B)
  std::unique_ptr<struct ResNet> rn;
};

// `stop_after` (test hook dg_emb_debug_stage): -1 returns before TDNN1, L after TDNN layer L (0-based)
int emb_trunk(dg_emb* h, const float* wav, int U, const Geom& g, cudaStream_t st, int* T_out, bool defer_last,
              const SincPrep* prep, int stop_after = 99);
bool pool_fusable(const dg_emb* h, int K, const Geom& g);
int emb_tail(dg_emb* h, int B, const Geom& g, const float* weights, int F, int K, int T, bool fuse, int normalize, float norm,
             float* out, cudaStream_t st, int sm_cap = 0);
int emb_tail_sets(dg_emb* h, int B, const Geom& g, const float* weights /*[G][B][F][K]*/, int G, int F, int K, int T, bool fuse,
                  float* out, int64_t out_stride, cudaStream_t st, int sm_cap = 0);

// ==================================================================================== clustering (api_cluster.cu)
struct dg_cluster {
  int device = 0;
  ClusterParams p;
  DevBuf centers, active, init, prep, prep_d, record;
  DevBuf base, base_active, relabel;   // shared-identity mode: table at the last merge, relabel of created centres
};

// ================================================================================== resampling (api_stream.cu)
struct dg_resample {
  int device = 0;
  RsGeom g{};
  DevBuf taps;   // [n][T]
};

// ==================================================================================== gallery (api_gallery.cu)
// entries E [Gp][Dp] float64, zero padded (gallery.cu), norms En [G]; ws_*: the workspace of dg_gallery_query (its tables
// in one copy, the split partials)
struct dg_gallery {
  int device = 0, G = 0, Gp = 0, D = 0, Dp = 0;
  DevBuf E, En, ws_in, ws_d, ws_e;
};

// ======================================================================== device-side audio stream (api_stream.cu)
// rearrange_audio_stream (reference src/diart/operators.py:44-100) on the device: the host pushes each sample ONCE
// (8 000 new samples per chunk instead of the 80 000 of a stacked window: 8.2 MB instead of 82 MB per 256-chunk step),
// windows are formed from a circular ring in HBM.
struct dg_stream {
  int device = 0, S = 0, hop = 0, C = 0;   // S, hop, C and the counters are in samples at the source rate
  long long wpos = 0, rpos = 0;          // absolute sample counters: pushed / start of the next window
  dg_resample* rs = nullptr;             // borrowed; windows are resampled to rs's rate (dg_stream_create_resampled)
  DevBuf ring, ys, crop_items, crop_out; // ys: stream-form outputs of the last batch; crop_*: dg_stream_crop_host
  PinnedBuf crop_pin;
  PinnedBuf pin;                         // pinned mirror of the ring (staging for the uploads)
  Stream st;                             // uploads
  Event e_up, e_read;
  // uploads still reading the pinned mirror: (first absolute sample, event); a region of the mirror is rewritten only
  // after the upload that last used it has completed
  std::deque<std::pair<long long, Event>> inflight;
  std::vector<Event> spare;
};

int stream_window_len(const dg_stream* h);
int stream_expand(dg_stream* h, int B, float* wav_dev, cudaStream_t st);

// =============================================================================== device post-path (api_post.cu)
// DelayedAggregation (hamming, loose) + Binarize of reference diarization.py:205-232 on the device (post.cu).  The handle keeps
// the scores and speaker maps of the last `num_windows - 1` chunks (the reference's pred_buffer) on the device.
struct dg_post {
  int device = 0, F = 0, K = 0, M = 0, nw = 1;
  double tau = 0.5;
  DevBuf hamming, hist_seg, hist_map, in, header, turns, total;   // history [2][nw - 1] (copy `cur` holds n_hist chunks)
  int cur = 0, n_hist = 0, cap_B = 0;
  int turn_cap = 0;
  PinnedBuf pin;                  // pinned staging: tau, slot, rows and plan in, header + total + turn prefix out
};

// The plan rows every post-path launch (post.cu, vad.cu) relies on, checked on the host before any launch.  Row `row` at pl
// [4 + nw] aggregates 1 <= nb <= min(nw, before + 1) buffers, `before` being the chunks of its stream or file ahead of it (none
// is read before the first), over nf >= 1 frames with first_nf >= 0, into at most min(F + 1, 1023) output frames (the first
// chunk of a stream emits up to F + 1, which the post kernels' shared memory holds; a turn's frame fields have 10 bits).
int check_plan_row(const char* who, const int32_t* pl, int row, int nw, int before, int F);
// the B plan rows of a dg_post step, after the n_hist chunks of its history
int post_check(const char* who, const dg_post* h, int B, const int32_t* plan_host);
// the most turns B chunks of M speakers can emit: up to F + 1 output frames, every second one starting a turn
inline int post_turn_cap(int B, int M, int F) { return B * M * ((F + 2) / 2); }

int post_enqueue(dg_post* h, const float* seg_dev, const int32_t* map_dev, int B, const int32_t* plan_host, cudaStream_t st);
int post_finish(dg_post* h, int B, int32_t* header_host, uint32_t* turns_host, int turn_cap_host, int* n_turns,
                cudaStream_t st);

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
int download_turns(const char* who, const unsigned char* pin, const TurnOut& lay, const uint32_t* turns_dev,
                   int32_t* header_host, uint32_t* turns_host, int turn_cap_host, int* n_turns, cudaStream_t st);

// ============================================================================ network pass (api_pipeline.cu)
// a step's outputs: scores [B, F, K], embeddings [B, K, D], speaker maps [B, K], permuted scores [B, F, M]
struct StepShape {
  int B = 0, F = 0, K = 0;
  size_t seg_bytes() const { return (size_t)B * F * K * 4; }
  size_t emb_bytes(int D) const { return (size_t)B * K * D * 4; }
  size_t map_bytes() const { return (size_t)B * K * 4; }
  size_t permuted_bytes(int M) const { return (size_t)B * F * M * 4; }
};

// What the networks of a step use besides its batch and outputs: the model handles, the overlapped-speech penalty, and per
// scratch lane a segmentation stream, the front-end state, the OSP weights and two events; the embedding stream.  A dg_pipeline
// is one; a dg_multi owns another over the same model handles (the lane guards order their uses).
struct NetLanes {
  dg_seg* seg = nullptr;
  dg_emb* emb = nullptr;
  float gamma = 3.f, beta = 10.f;
  int normalize_weights = 0;
  int hop = 0;          // samples between consecutive windows of a batch (hint, dg_pipeline_set_hop); 0 = unknown
  DevBuf osp[2];
  SincPrep prep[2];
  Stream s_seg[2], s_emb;
  Event e_osp[2], e_prep[2], e_emb;
};

// creates the streams and events of `n` (segmentation streams at high priority, the embedding stream at low priority)
int net_lanes_create(NetLanes& n);
// segmentation chain on s_seg[lane] and embedding chain on s_emb, both starting after `start`; on return e_emb (recorded on
// s_emb) marks seg, osp and emb complete.  stream_hop > 0: the batch is windows of one stream that many samples apart.
// sets (or null: the handle's own gamma, beta, normalize): the OSP weights and embeddings of G sets over one trunk pass, set g's
// embeddings at emb + g emb_stride.
int pipeline_nets(NetLanes* h, const float* wav, int S, const StepShape& sh, float* seg, float* emb, cudaEvent_t start,
                  int lane, int stream_hop, const OspSets* sets = nullptr, int G = 1, int64_t emb_stride = 0);
