// The fused pipeline (dg_pipeline_*): synchronous and submitted steps, the whole-call entry points and the shared-identity
// exchange.
#include <math.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <atomic>
#include <chrono>
#include <condition_variable>
#include <functional>
#include <memory>
#include <mutex>
#include <thread>
#include <vector>

#include "host.cuh"

// ================================================================================ fused pipeline
// Persistent worker threads for the host-side gather of dg_pipeline_call_host (B separate pageable windows -> pinned staging):
// created once per pipeline handle; a job is one callable that every worker runs concurrently (the callable hands out work
// items through its own atomic counter).
class GatherPool {
 public:
  explicit GatherPool(int n) {
    for (int i = 0; i < n; i++) th_.emplace_back([this] { loop(); });
  }
  ~GatherPool() {
    {
      std::lock_guard<std::mutex> lk(mu_);
      stop_ = true;
    }
    cv_.notify_all();
    for (auto& t : th_) t.join();
  }
  int size() const { return (int)th_.size(); }
  void start(std::function<void()> fn) {       // returns at once; wait() returns when every worker has finished fn
    {
      std::lock_guard<std::mutex> lk(mu_);
      job_ = std::move(fn);
      generation_++;
      active_ = (int)th_.size();
    }
    cv_.notify_all();
  }
  void wait() {
    std::unique_lock<std::mutex> lk(mu_);
    done_.wait(lk, [this] { return active_ == 0; });
  }

 private:
  void loop() {
    int seen = 0;
    for (;;) {
      std::function<void()> fn;
      {
        std::unique_lock<std::mutex> lk(mu_);
        cv_.wait(lk, [&] { return stop_ || generation_ != seen; });
        if (stop_) return;
        seen = generation_;
        fn = job_;
      }
      fn();
      {
        std::lock_guard<std::mutex> lk(mu_);
        if (--active_ == 0) done_.notify_all();
      }
    }
  }
  std::vector<std::thread> th_;
  std::mutex mu_;
  std::condition_variable cv_, done_;
  std::function<void()> job_;
  int generation_ = 0, active_ = 0;
  bool stop_ = false;
};

struct StepOut { float *seg, *emb; int32_t* map; float* permuted; };   // where a step's outputs are or go; null: not wanted

// The networks' model handles, lanes and streams are the NetLanes base (host.cuh).
struct dg_pipeline : NetLanes {
  dg_cluster* clu;
  // Members are destroyed in reverse order: the streams and events (declared last) first, then the pinned staging, then
  // the device buffers and worker threads; the NetLanes base goes last.
  DevBuf wav, segd, embd, mapd, permd;
  // Every step runs through pipeline_enqueue.  Submitted step n (up to DG_MAX_INFLIGHT outstanding) uses result / input slot
  // n % 3 and scratch lane n & 1: two steps compute concurrently while the host uploads step n+2.  Synchronous steps use lane
  // 0 and the caller's buffers or wav / segd / ..., never a slot (collected pointers stay valid), and do not count in next_step.
  DevBuf slot_wav[3], slot_seg[3], slot_emb[3], slot_map[3];
  StepShape slot_shape[3];
  int outstanding = 0;
  long long next_step = 0;
  long long nets_calls = 0;             // dg_pipeline_nets_sets calls: call n runs on scratch lane n & 1
  long long ident_merged_upto = 0;      // steps below this index have had their maps relabelled by a merge
  std::unique_ptr<GatherPool> gather;   // worker threads of the host gather (created at the first dg_pipeline_call_host)
  DevBuf call_stream;                   // device image of the stream a dg_pipeline_call_host batch was cut from
  long long call_h2d_bytes = 0;         // bytes the last dg_pipeline_call_host uploaded
  PinnedBuf pin_wav;                    // pinned staging of dg_pipeline_call_host (B separate host windows -> one upload)
  Stream st, s_clu, s_h2d, s_d2h;
  Event e_start, e_done;
  Event e_h2d[3], e_slot_done[3], e_lane_done[2];
  // shared-identity mode inside the pipelined flow: export / merge run on the clustering stream, in order with the clustering
  // of the submitted steps, so the networks of the next steps keep running meanwhile (created at the first export)
  Event e_ident, e_ident_in;
  StepOut slot_out(int s) const { return {slot_seg[s].as<float>(), slot_emb[s].as<float>(), slot_map[s].as<int32_t>()}; }
};

extern "C" int dg_pipeline_create(dg_seg* seg, dg_emb* emb, dg_cluster* clu, float gamma, float beta,
                                  int normalize_weights, dg_pipeline** out) {
  if (!seg || !emb || !clu || !out) {
    set_error("dg_pipeline_create: null handle");
    return DG_EINVAL;
  }
  if (seg->device != emb->device || seg->device != clu->device) {
    set_error("dg_pipeline_create: handles live on different devices");
    return DG_EINVAL;
  }
  if (clu->p.D != emb->D) {
    set_error("dg_pipeline_create: clustering dimension != embedding dimension");
    return DG_EINVAL;
  }
  std::unique_ptr<dg_pipeline> h(new dg_pipeline());
  h->seg = seg; h->emb = emb; h->clu = clu;
  h->gamma = gamma; h->beta = beta; h->normalize_weights = normalize_weights;
  DG_CUDA(cudaSetDevice(seg->device));
  int lo = 0, hi = 0;
  DG_CUDA(cudaDeviceGetStreamPriorityRange(&lo, &hi));
  if (net_lanes_create(*h) || h->st.create() || h->s_clu.create(hi) || h->s_h2d.create() || h->s_d2h.create()) return DG_ECUDA;
  for (Event* e : {&h->e_start, &h->e_done, &h->e_h2d[0], &h->e_h2d[1], &h->e_h2d[2], &h->e_slot_done[0], &h->e_slot_done[1],
                   &h->e_slot_done[2], &h->e_lane_done[0], &h->e_lane_done[1]})
    if (e->create()) return DG_ECUDA;
  *out = h.release();
  return DG_OK;
}

// two-stream overlap inside a step: the segmentation chain (critical path, high priority) and the embedding trunk
// (independent of it until the pooling weights exist) run concurrently
int net_lanes_create(NetLanes& n) {
  int lo = 0, hi = 0;
  DG_CUDA(cudaDeviceGetStreamPriorityRange(&lo, &hi));
  if (n.s_seg[0].create(hi) || n.s_seg[1].create(hi) || n.s_emb.create(lo)) return DG_ECUDA;
  for (Event* e : {&n.e_osp[0], &n.e_osp[1], &n.e_prep[0], &n.e_prep[1], &n.e_emb})
    if (e->create()) return DG_ECUDA;
  DG_CUDA(cudaEventRecord(n.e_emb, n.s_emb));   // so that the first step's wait on it is well defined
  return DG_OK;
}

// DG_CALL_TIMING=1: device time stamps of the sub-batches of dg_pipeline_call_host (diagnostic)
struct CallDiag {
  cudaEvent_t t0 = nullptr, up[3], prep[3], trunk[3], seg[3], emb[3], clu[3];
  int j = 0;
  void create() {
    if (t0) return;
    cudaEventCreate(&t0);
    for (int i = 0; i < 3; i++)
      for (cudaEvent_t* e : {&up[i], &prep[i], &trunk[i], &seg[i], &emb[i], &clu[i]}) cudaEventCreate(e);
  }
};
static thread_local CallDiag* g_diag = nullptr;
#define DG_DIAG(field, stream)                                        \
  do {                                                                \
    if (g_diag) cudaEventRecord(g_diag->field[g_diag->j], stream);    \
  } while (0)

// grid cap of the embedding stream's persistent kernels while the segmentation stream runs a recurrence over B windows: the
// SMs the recurrence leaves free, or no cap if that would be half of the device or less
static int emb_sm_cap(int device, int B) {
  int sms = 132;
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device);
  const int lstm_ctas = lstm_tc_ctas(B);
  return sms - lstm_ctas > sms / 2 ? sms - lstm_ctas : 0;
}

int pipeline_nets(NetLanes* h, const float* wav, int S, const StepShape& sh, float* seg, float* emb, cudaEvent_t start,
                  int lane, int stream_hop, const OspSets* sets, int G, int64_t emb_stride) {
  int rc;
  const int B = sh.B, F = sh.F, K = sh.K;
  const Geom g = make_geom(S);
  // lane 0 / 1: segmentation stream, scratch set, OSP buffer and event of this step (consecutive pipelined steps
  // alternate, so step i+1's segmentation chain can start while step i's is still in its recurrence)
  cudaStream_t s_seg = h->s_seg[lane];
  DevBuf& osp = h->osp[lane];
  if (osp.ensure(sh.seg_bytes() * (sets ? G : 1))) return DG_ECUDA;
  DG_CUDA(cudaStreamWaitEvent(s_seg, start, 0));
  DG_CUDA(cudaStreamWaitEvent(h->s_emb, start, 0));
  // another pipeline (or a block-level call) that used these model handles' scratch last: stream-ordered hand-over
  LaneUse seg_use(h->seg->guard[lane], h, s_seg), emb_use(h->emb->guard, h, h->s_emb);
  if ((rc = seg_use.rc) || (rc = emb_use.rc)) return rc;
  // waveform statistics + standardised fp16 planes once, for both networks' SincNets
  SincPrep& prep = h->prep[lane];
  if ((rc = run_sinc_prep(prep, wav, B, g, s_seg, stream_hop ? stream_hop : h->hop, stream_hop != 0))) return rc;
  DG_CUDA(cudaEventRecord(h->e_prep[lane], s_seg));
  DG_DIAG(prep, s_seg);
  DG_CUDA(cudaStreamWaitEvent(h->s_emb, h->e_prep[lane], 0));
  // embedding trunk first in host order (low-priority stream, grid capped to the SMs the LSTM leaves free)
  int T = 0;
  const bool fuse = pool_fusable(h->emb, K, g);
  const int sm_cap = emb_sm_cap(h->seg->device, B);
  {
    SmLimit cap(sm_cap);
    if ((rc = emb_trunk(h->emb, wav, B, g, h->s_emb, &T, fuse, &prep))) return rc;
  }
  DG_DIAG(trunk, h->s_emb);
  if ((rc = seg_forward_lane(h->seg, lane, &prep, wav, B, S, seg, s_seg))) return rc;
  if (sets) rc = launch_osp_sets(seg, B, F, K, *sets, G, osp.as<float>(), s_seg);
  else rc = dg_osp(seg, B, F, K, h->gamma, h->beta, h->normalize_weights, osp.as<float>(), s_seg);
  if (rc) return rc;
  DG_CUDA(cudaEventRecord(h->e_osp[lane], s_seg));
  if ((rc = seg_use.end())) return rc;
  DG_DIAG(seg, s_seg);
  DG_CUDA(cudaStreamWaitEvent(h->s_emb, h->e_osp[lane], 0));
  // a fused TDNN5 needs the pooling weights: it runs here, after the segmentation of this step, with its grid capped like the
  // trunk's (the other lane's recurrence may hold lstm_tc_ctas(B) SMs at this point)
  if (sets) rc = emb_tail_sets(h->emb, B, g, osp.as<float>(), G, F, K, T, fuse, emb, emb_stride, h->s_emb, sm_cap);
  else rc = emb_tail(h->emb, B, g, osp.as<float>(), F, K, T, fuse, 1, 1.f, emb, h->s_emb, sm_cap);
  if (rc) return rc;
  DG_CUDA(cudaEventRecord(h->e_emb, h->s_emb));
  DG_DIAG(emb, h->s_emb);
  return emb_use.end();
}

extern "C" int dg_pipeline_set_hop(dg_pipeline* h, int hop_samples) {
  if (!h || hop_samples < 0) {
    set_error("dg_pipeline_set_hop: bad arguments");
    return DG_EINVAL;
  }
  h->hop = hop_samples;
  return DG_OK;
}

// Enqueues one step: networks on scratch lane `lane` after `start`, clustering on s_clu, outputs to `out`.  stream_hop > 0:
// the batch was cut on the device from one stream, windows that many samples apart (sinc layer in stream form, no overlap
// check).  slot >= 0: a submitted step in that result slot, marked clustered by e_slot_done[slot]; else by e_done.
static int pipeline_enqueue(dg_pipeline* h, const float* wav, int S, const StepShape& sh, int lane, cudaEvent_t start,
                            int stream_hop, const StepOut& out, int slot) {
  int rc;
  // the slot's previous occupant (three submits ago) must be fully clustered, and the lane's previous user past its
  // embeddings, before their buffers are rewritten
  for (cudaStream_t s : {(cudaStream_t)h->s_seg[lane], (cudaStream_t)h->s_emb}) {
    if (slot >= 0) DG_CUDA(cudaStreamWaitEvent(s, h->e_slot_done[slot], 0));
    DG_CUDA(cudaStreamWaitEvent(s, h->e_lane_done[lane], 0));
  }
  if ((rc = pipeline_nets(h, wav, S, sh, out.seg, out.emb, start, lane, stream_hop))) return rc;
  // the lane's scratch (waveform planes, segmentation activations, OSP weights) is free as soon as this step's embeddings
  // exist -- the clustering reads only the step's outputs -- so the step after next may start before this one is clustered
  DG_CUDA(cudaEventRecord(h->e_lane_done[lane], h->s_emb));
  DG_CUDA(cudaStreamWaitEvent(h->s_clu, h->e_emb, 0));
  if ((rc = dg_cluster_step(h->clu, out.seg, out.emb, sh.B, sh.F, sh.K, out.map, out.permuted, h->s_clu))) return rc;
  DG_CUDA(cudaEventRecord(slot >= 0 ? h->e_slot_done[slot] : h->e_done, h->s_clu));
  DG_DIAG(clu, h->s_clu);
  return DG_OK;
}

// a synchronous step: lane 0, no slot; `st` waits for its clustering
static int pipeline_step(dg_pipeline* h, const float* wav, int S, const StepShape& sh, const StepOut& out, cudaStream_t st,
                         int stream_hop) {
  int rc;
  // DG_NO_OVERLAP=1 (diagnostic): the networks and the clustering back to back on `st`, for kernel-alone timings
  static const bool serial = getenv("DG_NO_OVERLAP") && getenv("DG_NO_OVERLAP")[0] == '1';
  if (serial) {
    if (h->osp[0].ensure(sh.seg_bytes())) return DG_ECUDA;
    if ((rc = dg_seg_forward(h->seg, wav, sh.B, S, out.seg, st))) return rc;
    if ((rc = dg_osp(out.seg, sh.B, sh.F, sh.K, h->gamma, h->beta, h->normalize_weights, h->osp[0].as<float>(), st))) return rc;
    if ((rc = dg_emb_forward(h->emb, wav, h->osp[0].as<float>(), sh.B, S, sh.F, sh.K, 1, 1.f, out.emb, st))) return rc;
    return dg_cluster_step(h->clu, out.seg, out.emb, sh.B, sh.F, sh.K, out.map, out.permuted, st);
  }
  DG_CUDA(cudaSetDevice(h->seg->device));
  DG_CUDA(cudaEventRecord(h->e_start, st));
  if ((rc = pipeline_enqueue(h, wav, S, sh, 0, h->e_start, stream_hop, out, -1))) return rc;
  DG_CUDA(cudaStreamWaitEvent(st, h->e_done, 0));
  return DG_OK;
}

// `st` waits for `done` (if any), then copies the outputs of a step of shape `sh` from `src` to the non-null members of `dst`
static int copy_out(const dg_pipeline* h, cudaStream_t st, cudaEvent_t done, const StepShape& sh, const StepOut& src,
                    const StepOut& dst, cudaMemcpyKind kind) {
  if (done) DG_CUDA(cudaStreamWaitEvent(st, done, 0));
  if (dst.seg) DG_CUDA(cudaMemcpyAsync(dst.seg, src.seg, sh.seg_bytes(), kind, st));
  if (dst.emb) DG_CUDA(cudaMemcpyAsync(dst.emb, src.emb, sh.emb_bytes(h->emb->D), kind, st));
  if (dst.map) DG_CUDA(cudaMemcpyAsync(dst.map, src.map, sh.map_bytes(), kind, st));
  if (dst.permuted) DG_CUDA(cudaMemcpyAsync(dst.permuted, src.permuted, sh.permuted_bytes(h->clu->p.M), kind, st));
  return DG_OK;
}

extern "C" int dg_pipeline_step(dg_pipeline* h, const float* wav, int B, int S, float* seg, float* emb, int32_t* map,
                                float* permuted, void* stream) {
  if (!h || !wav || !seg || !emb || !map || B < 1) {
    set_error("dg_pipeline_step: bad arguments");
    return DG_EINVAL;
  }
  if (h->outstanding) {
    set_error("dg_pipeline_step: submitted steps are outstanding; collect them first");
    return DG_EINVAL;
  }
  int rc, F = 0, K = 0;
  if ((rc = dg_seg_dims(h->seg, S, &F, &K))) return rc;
  return pipeline_step(h, wav, S, {B, F, K}, {seg, emb, map, permuted}, (cudaStream_t)stream, 0);
}

// ---- pipelined variants (up to three steps outstanding, two computing): the sequential clustering of step i and the host copies overlap the
//      networks of step i+1.  Per stream the chunk order is preserved: clustering runs on one stream.
static const int DG_MAX_INFLIGHT = 3;

// enqueues submitted step next_step (result slot `slot` = next_step % 3, lane next_step & 1) and books it outstanding
static int pipeline_submit(dg_pipeline* h, int slot, const float* wav, int S, const StepShape& sh, cudaEvent_t start,
                           int stream_hop) {
  int rc;
  if (h->slot_seg[slot].ensure(sh.seg_bytes()) || h->slot_emb[slot].ensure(sh.emb_bytes(h->emb->D)) ||
      h->slot_map[slot].ensure(sh.map_bytes()))
    return DG_ECUDA;
  if ((rc = pipeline_enqueue(h, wav, S, sh, (int)(h->next_step & 1), start, stream_hop, h->slot_out(slot), slot))) return rc;
  h->slot_shape[slot] = sh;
  h->next_step++;
  h->outstanding++;
  return DG_OK;
}

// A submitted step whose windows are staged in its slot's input buffer: refused when DG_MAX_INFLIGHT steps are outstanding
// (`who` names the entry point); else s_h2d waits until the slot's previous occupant is clustered, fill(dst, &stream_hop)
// writes the [B, S] windows to dst on s_h2d (stream_hop: see pipeline_enqueue), and the step starts behind them.
template <class Fill>
static int submit_staged(dg_pipeline* h, const char* who, int S, const StepShape& sh, Fill&& fill) {
  if (h->outstanding >= DG_MAX_INFLIGHT) {
    set_error(std::string(who) + ": three steps are already outstanding; collect one first");
    return DG_EINVAL;
  }
  const int slot = (int)(h->next_step % 3);
  if (h->slot_wav[slot].ensure((size_t)sh.B * S * 4)) return DG_ECUDA;
  DG_CUDA(cudaStreamWaitEvent(h->s_h2d, h->e_slot_done[slot], 0));
  int rc, stream_hop = 0;
  if ((rc = fill(h->slot_wav[slot].as<float>(), &stream_hop))) return rc;
  DG_CUDA(cudaEventRecord(h->e_h2d[slot], h->s_h2d));
  DG_DIAG(up, h->s_h2d);
  return pipeline_submit(h, slot, h->slot_wav[slot].as<float>(), S, sh, h->e_h2d[slot], stream_hop);
}

extern "C" int dg_pipeline_submit(dg_pipeline* h, const float* wav_dev, int B, int S, void* stream) {
  if (!h || !wav_dev || B < 1) {
    set_error("dg_pipeline_submit: bad arguments");
    return DG_EINVAL;
  }
  if (h->outstanding >= DG_MAX_INFLIGHT) {
    set_error("dg_pipeline_submit: three steps are already outstanding; collect one first");
    return DG_EINVAL;
  }
  int rc, F = 0, K = 0;
  if ((rc = dg_seg_dims(h->seg, S, &F, &K))) return rc;
  DG_CUDA(cudaSetDevice(h->seg->device));
  DG_CUDA(cudaEventRecord(h->e_start, (cudaStream_t)stream));
  return pipeline_submit(h, (int)(h->next_step % 3), wav_dev, S, {B, F, K}, h->e_start, 0);
}

extern "C" int dg_pipeline_collect(dg_pipeline* h, const float** seg_dev, const float** emb_dev,
                                   const int32_t** map_dev, void* stream) {
  if (!h || h->outstanding < 1) {
    set_error("dg_pipeline_collect: nothing outstanding");
    return DG_EINVAL;
  }
  const int slot = (int)((h->next_step - h->outstanding) % 3);
  DG_CUDA(cudaStreamWaitEvent((cudaStream_t)stream, h->e_slot_done[slot], 0));
  if (seg_dev) *seg_dev = h->slot_seg[slot].as<float>();
  if (emb_dev) *emb_dev = h->slot_emb[slot].as<float>();
  if (map_dev) *map_dev = h->slot_map[slot].as<int32_t>();
  h->outstanding--;
  return DG_OK;
}

extern "C" int dg_pipeline_collect_copy(dg_pipeline* h, float* seg_dev, float* emb_dev, int32_t* map_dev,
                                        void* stream) {
  if (!h || h->outstanding < 1) {
    set_error("dg_pipeline_collect_copy: nothing outstanding");
    return DG_EINVAL;
  }
  const int slot = (int)((h->next_step - h->outstanding) % 3);
  const int rc = copy_out(h, (cudaStream_t)stream, h->e_slot_done[slot], h->slot_shape[slot], h->slot_out(slot),
                          {seg_dev, emb_dev, map_dev, nullptr}, cudaMemcpyDeviceToDevice);
  if (rc) return rc;
  h->outstanding--;
  return DG_OK;
}

extern "C" int dg_pipeline_submit_host(dg_pipeline* h, const float* wav_host, int B, int S) {
  if (!h || !wav_host || B < 1) {
    set_error("dg_pipeline_submit_host: bad arguments");
    return DG_EINVAL;
  }
  int rc, F = 0, K = 0;
  if ((rc = dg_seg_dims(h->seg, S, &F, &K))) return rc;
  DG_CUDA(cudaSetDevice(h->seg->device));
  return submit_staged(h, "dg_pipeline_submit_host", S, {B, F, K}, [&](float* dst, int*) {
    DG_CUDA(cudaMemcpyAsync(dst, wav_host, (size_t)B * S * 4, cudaMemcpyHostToDevice, h->s_h2d));
    return 0;
  });
}

extern "C" int dg_pipeline_collect_host(dg_pipeline* h, float* seg_host, float* emb_host, int32_t* map_host) {
  if (!h || h->outstanding < 1) {
    set_error("dg_pipeline_collect_host: nothing outstanding");
    return DG_EINVAL;
  }
  const int slot = (int)((h->next_step - h->outstanding) % 3);
  const int rc = copy_out(h, h->s_d2h, h->e_slot_done[slot], h->slot_shape[slot], h->slot_out(slot),
                          {seg_host, emb_host, map_host, nullptr}, cudaMemcpyDeviceToHost);
  if (rc) return rc;
  DG_CUDA(cudaStreamSynchronize(h->s_d2h));
  h->outstanding--;
  return DG_OK;
}

extern "C" int dg_pipeline_step_host(dg_pipeline* h, const float* wav_host, int B, int S, float* seg_host,
                                     float* emb_host, int32_t* map_host, float* permuted_host) {
  if (!h || !wav_host || B < 1) {
    set_error("dg_pipeline_step_host: bad arguments");
    return DG_EINVAL;
  }
  int rc;
  StepShape sh = {B};
  if ((rc = dg_seg_dims(h->seg, S, &sh.F, &sh.K))) return rc;
  DG_CUDA(cudaSetDevice(h->seg->device));
  if (h->wav.ensure((size_t)B * S * 4) || h->segd.ensure(sh.seg_bytes()) || h->embd.ensure(sh.emb_bytes(h->emb->D)) ||
      h->mapd.ensure(sh.map_bytes()) || (permuted_host && h->permd.ensure(sh.permuted_bytes(h->clu->p.M))))
    return DG_ECUDA;
  DG_CUDA(cudaMemcpyAsync(h->wav.p, wav_host, (size_t)B * S * 4, cudaMemcpyHostToDevice, h->st));
  const StepOut dev = {h->segd.as<float>(), h->embd.as<float>(), h->mapd.as<int32_t>(),
                       permuted_host ? h->permd.as<float>() : nullptr};
  if ((rc = dg_pipeline_step(h, h->wav.as<float>(), B, S, dev.seg, dev.emb, dev.map, dev.permuted, h->st))) return rc;
  if ((rc = copy_out(h, h->st, nullptr, sh, dev, {seg_host, emb_host, map_host, permuted_host}, cudaMemcpyDeviceToHost)))
    return rc;
  DG_CUDA(cudaStreamSynchronize(h->st));
  return DG_OK;
}

// worker threads of the host gather, created at the first dg_pipeline_call_host: all cores but two, at most 24
static GatherPool& gather_pool(dg_pipeline* h) {
  if (!h->gather) h->gather.reset(new GatherPool(std::max(1, std::min((int)std::thread::hardware_concurrency() - 2, 24))));
  return *h->gather;
}

// ---- the whole body of SpeakerDiarization.__call__ (reference diarization.py:172-232) in one call: B separate host windows
//      (as rearrange_audio_stream emits them) are gathered into pinned staging by worker threads while earlier rows are
//      already on their way to the device, then fused step + post-path, one D2H of the turn list.
static int upload_rows(dg_pipeline* h, const float* const* rows, int B, int S, float* pin, float* dst_dev, cudaStream_t st) {
  const int R = 4;                                    // rows per work item (1.3 MB at S = 80000)
  const int items = (B + R - 1) / R;
  GatherPool& pool = gather_pool(h);
  std::vector<std::atomic<int>> done(items);
  for (auto& d : done) d.store(0, std::memory_order_relaxed);
  std::atomic<int> next{0};
  pool.start([&]() {
    for (;;) {
      const int it = next.fetch_add(1, std::memory_order_relaxed);
      if (it >= items) return;
      const int r0 = it * R, r1 = std::min(B, r0 + R);
      for (int r = r0; r < r1; r++) memcpy(pin + (size_t)r * S, rows[r], (size_t)S * 4);
      done[it].store(1, std::memory_order_release);
    }
  });
  // the calling thread forwards finished items, in order, in runs of up to 8 (~10 MB per copy)
  cudaError_t err = cudaSuccess;
  int sent = 0;
  while (sent < items) {
    int upto = sent;
    while (upto < items && upto - sent < 8 && done[upto].load(std::memory_order_acquire)) upto++;
    if (upto == sent) {
      std::this_thread::yield();
      continue;
    }
    const int r0 = sent * R, r1 = std::min(B, upto * R);
    if (err == cudaSuccess)
      err = cudaMemcpyAsync(dst_dev + (size_t)r0 * S, pin + (size_t)r0 * S, (size_t)(r1 - r0) * S * 4, cudaMemcpyHostToDevice, st);
    sent = upto;
  }
  pool.wait();          // (`next` and `done` live on this frame)
  DG_CUDA(err);
  return 0;
}

// Windows that are consecutive hops of ONE stream -- what the reference's rearrange_audio_stream emits (operators.py:44-100) --
// share S - hop samples with their neighbour.  The workers compare every window with its predecessor (memcmp of the shared
// samples, exact) and pack the `hop` new samples of each into the pinned stream image; the caller then uploads
// S + (B - 1) hop samples instead of B S and forms the windows on the device.  Returns 1 if windows [r0, r0 + nb) continue the
// stream (pin_stream[0 .. S + (r0 + nb - 1) hop) is then valid), 0 if some window does not (the caller falls back to the
// full gather for this and the following sub-batches).
static int pack_stream_rows(dg_pipeline* h, const float* const* rows, int r0, int nb, int S, int hop, float* pin_stream) {
  GatherPool& pool = gather_pool(h);
  std::atomic<int> next{r0}, bad{0};
  pool.start([&]() {
    for (;;) {
      const int r = next.fetch_add(1, std::memory_order_relaxed);
      if (r >= r0 + nb || bad.load(std::memory_order_relaxed)) return;
      if (r == 0) {
        memcpy(pin_stream, rows[0], (size_t)S * 4);
      } else if (memcmp(rows[r - 1] + hop, rows[r], (size_t)(S - hop) * 4) != 0) {
        bad.store(1, std::memory_order_relaxed);
      } else {
        memcpy(pin_stream + (size_t)S + (size_t)(r - 1) * hop, rows[r] + (S - hop), (size_t)hop * 4);
      }
    }
  });
  pool.wait();
  return bad.load() ? 0 : 1;
}

static bool post_fits(const dg_pipeline* h, const dg_post* post, const StepShape& sh) {
  return sh.F == post->F && sh.K == post->K && h->clu->p.M == post->M && post->device == h->seg->device;
}

// end of dg_pipeline_call_host / _call_stream, with the batch's scores and maps in segd / mapd (ordered on h->st) and the plan
// rows checked at entry (post_check): post-path, optional downloads, one synchronise (time stamp in *synced, if given), turn list
static int call_finish(dg_pipeline* h, dg_post* post, const StepShape& sh, const int32_t* plan_host, int32_t* header_host,
                       uint32_t* turns_host, int turn_cap_host, int* n_turns, float* seg_host, int32_t* map_host,
                       std::chrono::steady_clock::time_point* synced) {
  int rc;
  const StepOut dev = {h->segd.as<float>(), nullptr, h->mapd.as<int32_t>(), nullptr};
  if ((rc = post_enqueue(post, dev.seg, dev.map, sh.B, plan_host, h->st))) return rc;
  if ((rc = copy_out(h, h->st, nullptr, sh, dev, {seg_host, nullptr, map_host, nullptr}, cudaMemcpyDeviceToHost))) return rc;
  DG_CUDA(cudaStreamSynchronize(h->st));
  if (synced) *synced = std::chrono::steady_clock::now();
  return post_finish(post, sh.B, header_host, turns_host, turn_cap_host, n_turns, h->st);
}

extern "C" int dg_pipeline_call_host(dg_pipeline* h, dg_post* post, const float* const* rows_host, int B, int S,
                                     const int32_t* plan_host, int32_t* header_host, uint32_t* turns_host, int turn_cap_host,
                                     int* n_turns, float* seg_host, int32_t* map_host) {
  if (!h || !post || !rows_host || !plan_host || !header_host || !turns_host || B < 1) {
    set_error("dg_pipeline_call_host: bad arguments");
    return DG_EINVAL;
  }
  int rc;
  StepShape sh = {B};
  if ((rc = dg_seg_dims(h->seg, S, &sh.F, &sh.K))) return rc;
  if (!post_fits(h, post, sh)) {
    set_error("dg_pipeline_call_host: post handle was created for other dimensions");
    return DG_EINVAL;
  }
  if (h->outstanding) {
    set_error("dg_pipeline_call_host: submitted steps are outstanding; collect them first");
    return DG_EINVAL;
  }
  if ((rc = post_check("dg_pipeline_call_host", post, B, plan_host))) return rc;
  DG_CUDA(cudaSetDevice(h->seg->device));
  // DG_CALL_TIMING=1: host wall-clock phases of the call on stderr (diagnostic)
  static const bool call_timing = getenv("DG_CALL_TIMING") && getenv("DG_CALL_TIMING")[0] == '1';
  const auto tc0 = std::chrono::steady_clock::now();
  static thread_local CallDiag diag;
  if (call_timing) {
    diag.create();
    cudaEventRecord(diag.t0, h->s_h2d);
    g_diag = &diag;
  }
  if (h->segd.ensure(sh.seg_bytes()) || h->mapd.ensure(sh.map_bytes())) return DG_ECUDA;
  if (h->pin_wav.ensure((size_t)B * S * 4)) return DG_ECUDA;
  // The batch runs as up to three sub-batches through the pipelined machinery (dg_pipeline_submit_host): the upload of
  // sub-batch j+1 and its front end overlap the recurrence of sub-batch j; clustering stays in chunk order on its one stream,
  // so the result is exactly that of one step over the whole batch.  From 64 windows on: two halves; from 192 windows on:
  // three parts -- a short first one so that the device starts early and a short last one, because its dependent chain
  // (1172 recurrence steps + its share of the clustering) is what the caller waits for at the end
  int plan[DG_MAX_INFLIGHT] = {B, 0, 0}, ns = 1;
  if (B >= 192) {
    ns = 3;
    plan[0] = (B * 5 / 16 + 7) / 8 * 8;
    plan[2] = (B * 4 / 16 + 7) / 8 * 8;
    plan[1] = B - plan[0] - plan[2];
  } else if (B >= 64) {
    ns = 2;
    plan[0] = (B / 2 + 7) / 8 * 8;
    plan[1] = B - plan[0];
  }
  // consecutive windows of one stream (hop known from dg_pipeline_set_hop): verified on the host, uploaded once (see
  // pack_stream_rows)
  const int hop = h->hop;
  bool as_stream = hop > 0 && hop < S && hop % 4 == 0 && S % 4 == 0 && B >= 2;
  const size_t stream_len = (size_t)S + (size_t)(B - 1) * (hop > 0 ? hop : 0);
  if (as_stream && h->call_stream.ensure((stream_len + 64) * 4)) return DG_ECUDA;
  float* pin = h->pin_wav.as<float>();
  h->call_h2d_bytes = 0;
  for (int j = 0, r0 = 0; j < ns; r0 += plan[j], j++) {
    const int nb = plan[j];
    if (g_diag) g_diag->j = j;
    const auto fill = [&](float* dst, int* stream_hop) {
      if (as_stream && !pack_stream_rows(h, rows_host, r0, nb, S, hop, pin)) as_stream = false;
      if (as_stream) {
        // the samples this sub-batch adds to the device image of the stream, then its windows from that image
        const size_t lo = r0 == 0 ? 0 : (size_t)S + (size_t)(r0 - 1) * hop, hi = (size_t)S + (size_t)(r0 + nb - 1) * hop;
        DG_CUDA(cudaMemcpyAsync(h->call_stream.as<float>() + lo, pin + lo, (hi - lo) * 4, cudaMemcpyHostToDevice, h->s_h2d));
        h->call_h2d_bytes += (long long)(hi - lo) * 4;
        const long long cap = (long long)((stream_len + 3) / 4 * 4 + 4);     // linear image: the ring index never wraps
        *stream_hop = hop;
        return launch_expand_windows(h->call_stream.as<float>(), (long long)r0 * hop, (int)cap, hop, S, nb, dst, h->s_h2d);
      }
      // (after a failed stream check the pinned buffer is reused as the [B, S] staging: earlier sub-batches are already on the device)
      if (h->call_h2d_bytes) DG_CUDA(cudaStreamSynchronize(h->s_h2d));
      if ((rc = upload_rows(h, rows_host + r0, nb, S, pin + (size_t)r0 * S, dst, h->s_h2d))) return rc;
      h->call_h2d_bytes += (long long)nb * S * 4;
      return 0;
    };
    if ((rc = submit_staged(h, "dg_pipeline_call_host", S, {nb, sh.F, sh.K}, fill))) return rc;
  }
  for (int j = 0, r0 = 0; j < ns; r0 += plan[j], j++)     // collect the sub-batches' scores / maps, in order
    if ((rc = dg_pipeline_collect_copy(h, h->segd.as<float>() + (size_t)r0 * sh.F * sh.K, nullptr,
                                       h->mapd.as<int32_t>() + (size_t)r0 * sh.K, h->st)))
      return rc;
  const auto tc1 = std::chrono::steady_clock::now();
  auto tc2 = tc1;
  rc = call_finish(h, post, sh, plan_host, header_host, turns_host, turn_cap_host, n_turns, seg_host, map_host, &tc2);
  g_diag = nullptr;
  if (call_timing) {
    static int shown = 0;
    if (rc == 0 && shown++ % 4 == 3) {
      for (int j = 0; j < ns; j++) {
        float t[6] = {0, 0, 0, 0, 0, 0};
        cudaEvent_t ev[6] = {diag.up[j], diag.prep[j], diag.trunk[j], diag.seg[j], diag.emb[j], diag.clu[j]};
        for (int q = 0; q < 6; q++) cudaEventElapsedTime(&t[q], diag.t0, ev[q]);
        fprintf(stderr, "  sub-batch %d (%d windows), ms after entry: uploaded %.2f | front end %.2f | embedding trunk %.2f | segmentation + "
                        "OSP %.2f | embeddings %.2f | clustered %.2f\n", j, plan[j], t[0], t[1], t[2], t[3], t[4], t[5]);
      }
    }
    static double acc[3] = {0, 0, 0};
    static int calls = 0;
    const auto ms = [](std::chrono::steady_clock::time_point a, std::chrono::steady_clock::time_point b) {
      return std::chrono::duration<double, std::milli>(b - a).count(); };
    acc[0] += ms(tc0, tc1);
    acc[1] += ms(tc1, tc2);
    acc[2] += ms(tc2, std::chrono::steady_clock::now());
    if (++calls % 4 == 0) {
      fprintf(stderr, "dg_pipeline_call_host (B=%d, %d sub-batches): gather + upload + enqueue %.2f ms | wait for the device %.2f ms | "
                      "turn list %.2f ms (mean of 4 calls)\n", B, ns, acc[0] / 4, acc[1] / 4, acc[2] / 4);
      acc[0] = acc[1] = acc[2] = 0;
    }
  }
  return rc;
}

extern "C" int64_t dg_pipeline_last_call_h2d_bytes(const dg_pipeline* h) { return h ? (int64_t)h->call_h2d_bytes : 0; }

// ---- shared-identity mode (SURVEY.md 8(e), BASELINE config 5) without leaving the pipelined flow.  After dg_pipeline_submit*:
//   dg_pipeline_identity_export  enqueues the export of this rank's centroid changes behind the clustering of every submitted
//                                step (clustering stream) and makes `stream` wait for it -> the caller all-gathers the records
//   dg_pipeline_identity_merge   makes the clustering stream wait for `stream` (the all-gather), merges all ranks' records and
//                                relabels the speaker maps of the steps clustered since the previous merge (still on the device)
// The clustering of the NEXT submitted step is ordered behind the merge, exactly as in the one-step-at-a-time protocol; only
// the networks of the next steps overlap the exchange.  Call the pair once after every submit, before collecting that step.
extern "C" int dg_pipeline_identity_export(dg_pipeline* h, double* record_dev, void* stream) {
  if (!h || !record_dev) {
    set_error("dg_pipeline_identity_export: bad arguments");
    return DG_EINVAL;
  }
  DG_CUDA(cudaSetDevice(h->seg->device));
  if (!h->e_ident && (h->e_ident.create() || h->e_ident_in.create())) return DG_ECUDA;
  int rc;
  if ((rc = dg_cluster_export_delta(h->clu, record_dev, h->s_clu))) return rc;
  DG_CUDA(cudaEventRecord(h->e_ident, h->s_clu));
  DG_CUDA(cudaStreamWaitEvent((cudaStream_t)stream, h->e_ident, 0));
  return DG_OK;
}

extern "C" int dg_pipeline_identity_merge(dg_pipeline* h, const double* records_dev, int world, int rank, void* stream) {
  if (!h || !records_dev || world < 1 || rank < 0 || rank >= world || !h->e_ident) {
    set_error("dg_pipeline_identity_merge: bad arguments (or no export before it)");
    return DG_EINVAL;
  }
  DG_CUDA(cudaSetDevice(h->seg->device));
  DG_CUDA(cudaEventRecord(h->e_ident_in, (cudaStream_t)stream));
  DG_CUDA(cudaStreamWaitEvent(h->s_clu, h->e_ident_in, 0));
  int rc;
  long long first = h->ident_merged_upto;
  if (first < h->next_step - DG_MAX_INFLIGHT) first = h->next_step - DG_MAX_INFLIGHT;
  bool merged = false;
  for (long long step = first; step < h->next_step; step++) {
    const int slot = (int)(step % 3);
    int32_t* maps = h->slot_map[slot].as<int32_t>();
    const int n = h->slot_shape[slot].B * h->slot_shape[slot].K;
    if (!merged) {
      if ((rc = dg_cluster_merge(h->clu, records_dev, world, rank, maps, n, h->s_clu))) return rc;
      merged = true;
    } else if ((rc = launch_relabel_maps(maps, n, h->clu->relabel.as<int32_t>(), h->s_clu))) {
      return rc;
    }
    DG_CUDA(cudaEventRecord(h->e_slot_done[slot], h->s_clu));      // collect must see the relabelled maps
  }
  if (!merged && (rc = dg_cluster_merge(h->clu, records_dev, world, rank, nullptr, 0, h->s_clu))) return rc;
  h->ident_merged_upto = h->next_step;
  return DG_OK;
}

// pipelined step whose batch is the next B windows of a device-side stream (no window upload at all; the sinc layer takes
// its stream form without the overlap check: the windows overlap by construction)
extern "C" int dg_pipeline_submit_stream(dg_pipeline* h, dg_stream* s, int B) {
  if (!h || !s || B < 1) {
    set_error("dg_pipeline_submit_stream: bad arguments");
    return DG_EINVAL;
  }
  if (s->device != h->seg->device) {
    set_error("dg_pipeline_submit_stream: stream and pipeline live on different devices");
    return DG_EINVAL;
  }
  int rc, F = 0, K = 0;
  const int S = stream_window_len(s);
  if ((rc = dg_seg_dims(h->seg, S, &F, &K))) return rc;
  DG_CUDA(cudaSetDevice(h->seg->device));
  return submit_staged(h, "dg_pipeline_submit_stream", S, {B, F, K}, [&](float* dst, int* stream_hop) {
    // resampled windows differ from exact hops of one stream at their edges: no stream-form claim for them
    *stream_hop = s->rs ? 0 : s->hop;
    return stream_expand(s, B, dst, h->s_h2d);
  });
}

// SpeakerDiarization.__call__ for the next B windows of a device-side stream: fused step + post-path, synchronous
extern "C" int dg_pipeline_call_stream(dg_pipeline* h, dg_post* post, dg_stream* s, int B, const int32_t* plan_host,
                                       int32_t* header_host, uint32_t* turns_host, int turn_cap_host, int* n_turns,
                                       float* seg_host, int32_t* map_host) {
  if (!h || !post || !s || !plan_host || !header_host || !turns_host || B < 1) {
    set_error("dg_pipeline_call_stream: bad arguments");
    return DG_EINVAL;
  }
  if (h->outstanding) {
    set_error("dg_pipeline_call_stream: submitted steps are outstanding; collect them first");
    return DG_EINVAL;
  }
  int rc;
  const int S = stream_window_len(s);
  StepShape sh = {B};
  if ((rc = dg_seg_dims(h->seg, S, &sh.F, &sh.K))) return rc;
  if (!post_fits(h, post, sh) || s->device != h->seg->device) {
    set_error("dg_pipeline_call_stream: handles were created for other dimensions / devices");
    return DG_EINVAL;
  }
  if ((rc = post_check("dg_pipeline_call_stream", post, B, plan_host))) return rc;
  DG_CUDA(cudaSetDevice(h->seg->device));
  if (h->wav.ensure((size_t)B * S * 4) || h->segd.ensure(sh.seg_bytes()) || h->embd.ensure(sh.emb_bytes(h->emb->D)) ||
      h->mapd.ensure(sh.map_bytes()))
    return DG_ECUDA;
  if ((rc = stream_expand(s, B, h->wav.as<float>(), h->st))) return rc;
  const StepOut dev = {h->segd.as<float>(), h->embd.as<float>(), h->mapd.as<int32_t>(), nullptr};
  if ((rc = pipeline_step(h, h->wav.as<float>(), S, sh, dev, h->st, s->rs ? 0 : s->hop))) return rc;
  return call_finish(h, post, sh, plan_host, header_host, turns_host, turn_cap_host, n_turns, seg_host, map_host, nullptr);
}

// The networks of one batch without clustering, for G OSP sets: scores [B, F, K] to seg_dev and set g's embeddings [B, K, D] to
// emb_dev + g emb_set_stride.  Consecutive calls alternate the two scratch lanes like submitted steps, so the segmentation of
// call n + 1 overlaps the embedding tail of call n; `stream` waits for this call's outputs.  The sinc front end takes the form
// the hop hint (dg_pipeline_set_hop) selects, as in dg_pipeline_submit.
extern "C" int dg_pipeline_nets_sets(dg_pipeline* h, const float* wav_dev, int B, int S, int num_sets, const float* osp_host,
                                     const int32_t* normalize_host, float* seg_dev, float* emb_dev, int64_t emb_set_stride,
                                     void* stream) {
  const char* who = "dg_pipeline_nets_sets";
  if (!h || !wav_dev || !seg_dev || !emb_dev || !osp_host || !normalize_host || B < 1 || num_sets < 1 ||
      num_sets > DG_MAX_OSP_SETS) {
    set_error(std::string(who) + ": bad arguments (need B >= 1, 1 <= num_sets <= 64, non-null buffers)");
    return DG_EINVAL;
  }
  OspSets sets{};
  for (int g = 0; g < num_sets; g++) {
    sets.gamma[g] = osp_host[2 * g];
    sets.beta[g] = osp_host[2 * g + 1];
    sets.normalize[g] = normalize_host[g];
    if (!std::isfinite(sets.gamma[g]) || !std::isfinite(sets.beta[g]) || (unsigned)sets.normalize[g] > 1u) {
      set_error(std::string(who) + ": set " + std::to_string(g) + " needs finite gamma and beta and normalize 0 or 1");
      return DG_EINVAL;
    }
  }
  int rc, F = 0, K = 0;
  if ((rc = dg_seg_dims(h->seg, S, &F, &K))) return rc;
  const int64_t per_set = (int64_t)B * K * h->emb->D;
  if (num_sets > 1 && emb_set_stride < per_set) {
    set_error(std::string(who) + ": emb_set_stride " + std::to_string(emb_set_stride) + " is below one set's B K D = " +
              std::to_string(per_set));
    return DG_EINVAL;
  }
  if (h->outstanding) {
    set_error(std::string(who) + ": submitted steps are outstanding; collect them first");
    return DG_EINVAL;
  }
  DG_CUDA(cudaSetDevice(h->seg->device));
  const int lane = (int)(h->nets_calls & 1);
  DG_CUDA(cudaEventRecord(h->e_start, (cudaStream_t)stream));
  // the lane's previous user must be past its embeddings before its scratch is rewritten
  for (cudaStream_t s : {(cudaStream_t)h->s_seg[lane], (cudaStream_t)h->s_emb}) DG_CUDA(cudaStreamWaitEvent(s, h->e_lane_done[lane], 0));
  if ((rc = pipeline_nets(h, wav_dev, S, {B, F, K}, seg_dev, emb_dev, h->e_start, lane, 0, &sets, num_sets, emb_set_stride)))
    return rc;
  DG_CUDA(cudaEventRecord(h->e_lane_done[lane], h->s_emb));
  DG_CUDA(cudaStreamWaitEvent((cudaStream_t)stream, h->e_lane_done[lane], 0));
  h->nets_calls++;
  return DG_OK;
}

extern "C" int dg_pipeline_destroy(dg_pipeline* h) {
  delete h;
  return DG_OK;
}
