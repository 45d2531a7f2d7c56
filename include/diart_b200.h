/*
 * diart_b200 -- C ABI of the H100-native diart hot path (libdiartb200.so, sm_90a).
 *
 * This is the drop-in boundary (SURVEY.md section 8(b)).  The reference is pure Python and has
 * no FFI of its own; each entry point below names the reference interface it replaces and is
 * what a ctypes/cffi binding of that interface would call (see INTEGRATION.md).
 *
 * Conventions
 *   - every function returns 0 on success, a negative DG_E* code on failure; the message is
 *     available from dg_last_error() (thread-local).
 *   - pointers documented "dev" are device pointers on the handle's device; "host" are host
 *     pointers.  Device entry points are stream-ordered on `stream` (a cudaStream_t passed as
 *     void*, NULL = legacy default stream) and never synchronise, except where noted.
 *   - a handle is not thread-safe; distinct handles are independent.  This matches the
 *     reference, where a pipeline instance is only ever driven by one thread
 *     (reference src/diart/inference.py:230).
 *   - tensors are dense, row-major, float32 unless stated otherwise.
 */
#ifndef DIART_B200_H
#define DIART_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define DG_OK 0
#define DG_EINVAL (-1)   /* bad argument / shape (the reference raises AssertionError / ValueError) */
#define DG_ECUDA (-2)    /* CUDA runtime error */
#define DG_EWEIGHT (-3)  /* missing / mis-shaped tensor in the state dict */
#define DG_ENCCL (-4)

/* One named float32 tensor of a pyannote state_dict (host memory), e.g.
 * {"sincnet.conv1d.1.weight", ptr, 24000}.  Key names follow pyannote.audio's PyanNet /
 * XVectorSincNet modules -- what reference src/diart/models.py:50 loads. */
typedef struct dg_tensor {
  const char* name;
  const float* data;
  int64_t numel;
} dg_tensor;

typedef struct dg_seg dg_seg;
typedef struct dg_emb dg_emb;
typedef struct dg_cluster dg_cluster;
typedef struct dg_pipeline dg_pipeline;
typedef struct dg_post dg_post;
typedef struct dg_stream dg_stream;
typedef struct dg_sweep dg_sweep;
typedef struct dg_vad_sweep dg_vad_sweep;

const char* dg_last_error(void);
int dg_version(void);

/* ---- segmentation model: replaces the callable behind SegmentationModel.__call__
 *      (reference src/diart/models.py:188-198; call site src/diart/blocks/segmentation.py:47):
 *      waveform (B,1,S) -> (B,F,K) sigmoid scores. ---- */
int dg_seg_create(const dg_tensor* tensors, int n_tensors, int device, dg_seg** out);
/* frames / local speakers produced for `num_samples`-sample chunks (293 / 3 for 80000) */
int dg_seg_dims(const dg_seg* h, int num_samples, int* frames, int* speakers);
/* Powerset models (pyannote/segmentation-3.0; reference PowersetAdapter, src/diart/models.py:29-39): the classifier has
 * one output per subset of the `num_speakers` local speakers of size <= `max_per_frame` (pyannote Powerset order: by
 * size, then lexicographic); forward then returns the hard multilabel scores one_hot(argmax) @ mapping, (B, F,
 * num_speakers), and dg_seg_dims reports num_speakers. */
int dg_seg_set_powerset(dg_seg* h, int num_speakers, int max_per_frame);
int dg_seg_forward(dg_seg* h, const float* wav_dev /*[B,S]*/, int B, int S,
                   float* seg_dev /*[B,F,K]*/, void* stream);
int dg_seg_destroy(dg_seg* h);

/* ---- embedding model: replaces the callable behind EmbeddingModel.__call__
 *      (reference src/diart/models.py:248-265; call site src/diart/blocks/embedding.py:60-67).
 *      pool_mode: 31 = pyannote.audio 3.1 StatsPool (nearest resize, +1e-8), 21 = 2.1 (linear). ---- */
int dg_emb_create(const dg_tensor* tensors, int n_tensors, int pool_mode, int device, dg_emb** out);
int dg_emb_dims(const dg_emb* h, int num_samples, int* frames, int* dimension);
/* Fused form: one trunk pass per waveform, K weighted poolings.
 * weights_dev [B,F,K] (the layout OverlappedSpeechPenalty returns) or NULL (unweighted, K must be 1).
 * If normalize != 0 rows are L2-normalised to `norm` (EmbeddingNormalization,
 * reference src/diart/blocks/embedding.py:110-120).  out_dev [B,K,D]. */
int dg_emb_forward(dg_emb* h, const float* wav_dev /*[B,S]*/, const float* weights_dev, int B, int S,
                   int F, int K, int normalize, float norm, float* out_dev, void* stream);
/* Compatibility form, exactly the arguments the reference block passes
 * (src/diart/blocks/embedding.py:57-65): waveform rows already repeated K times, weights (N,F).
 * Consecutive identical waveform rows are detected on the device and share one trunk pass.
 * Performs one small D2H read (row-group flags), i.e. synchronises `stream`. */
int dg_emb_forward_rows(dg_emb* h, const float* wav_dev /*[N,S]*/, const float* weights_dev /*[N,F] or NULL*/,
                        int N, int S, int F, float* out_dev /*[N,D]*/, void* stream);
int dg_emb_destroy(dg_emb* h);
/* Variant B -- pyannote/wespeaker-voxceleb-resnet34-LM (reference README.md:172-173, loaded through src/diart/models.py:50,59):
 * dg_emb_create recognises the checkpoint by its key names (resnet.conv1.weight, resnet.layer1.0.conv1.weight, ...,
 * resnet.seg_1.weight) and every dg_emb_* entry point then runs kaldi fbank -> ResNet34 -> TSTP -> Linear(5120, 256);
 * chunk lengths must be multiples of 160 samples.  Test hook: the trunk up to the stem (stop_after = -1) or BasicBlock
 * stop_after (0..15), returned as float32 [U][W][H][C] (time, mel, channel) on the host; -2 = log-mel features [U][T][80].
 * dims receives {U, W, H, C}.  Synchronises the device. */
int dg_emb_debug_trunk(dg_emb* h, const float* wav_dev, int U, int S, int stop_after, float* out_host, int64_t cap, int* dims);
/* Test hooks of the default networks (PyanNet, XVectorSincNet): the production forward with a host-side stop point, and the
 * map it left on the device returned as float32 on the host -- un-padded rows, real channels, fp16 hi / lo planes as hi + lo.
 * hop > 0: the front end runs as under dg_pipeline_set_hop(hop) (stream form of the sinc layer when the device finds the batch
 * a run of overlapping windows); hop = 0: the per-window form.  Stages shared by both: 0 operand of conv1 [B][T0][80],
 * 1 operand of conv2 [B][T1][60], 2 operand of the LSTM / TDNN1 [B][T2][60], 3 waveform mean and rstd [2][B].
 * dg_seg_debug_stage: 4..7 output of LSTM layer 0..3 [B][T2][256], 8 / 9 the two Linears [B][T2][128], 10 scores [B][T2][K]
 * (powerset handles: the decoded {0, 1} labels [B][T2][num_speakers]).
 * dg_emb_debug_stage: 4..7 TDNN1..4 [B][T][512], 8 TDNN5 [B][T][1500], 9 / 10 pooled statistics [B*K][3000] from the fused /
 * un-fused pooling, 11 / 12 the raw embedding [B*K][D] behind either; weights_dev [B][F][K] is read from stage 9 on.
 * dims receives the three extents and, in dims[3], the paths taken: 1 stream form, 2 MaxPool1d(3) fused into conv1 / conv2,
 * 4 recurrence with 16 rows per CTA, 8 fused statistics pooling.  Both synchronise the device. */
int dg_seg_debug_stage(dg_seg* h, const float* wav_dev, int B, int S, int hop, int stage, float* out_host, int64_t cap, int* dims);
int dg_emb_debug_stage(dg_emb* h, const float* wav_dev, const float* weights_dev, int B, int S, int F, int K, int hop, int stage,
                       float* out_host, int64_t cap, int* dims);

/* ---- element-wise blocks ---- */
/* OverlappedSpeechPenalty (reference src/diart/blocks/embedding.py:98-107, functional.py:6-13) */
int dg_osp(const float* seg_dev /*[B,F,K]*/, int B, int F, int K, float gamma, float beta,
           int normalize, float* out_dev, void* stream);
/* EmbeddingNormalization (reference src/diart/functional.py:16-27): out = norm * e / ||e||_2 */
int dg_normalize_embeddings(const float* emb_dev /*[rows,D]*/, int rows, int D, float norm,
                            float* out_dev, void* stream);

/* ---- OnlineSpeakerClustering (reference src/diart/blocks/clustering.py:31-218 and the
 *      SpeakerMap logic of src/diart/mapping.py:179-360).  State (centroids, float64) lives on
 *      the device. ---- */
int dg_cluster_create(int max_speakers, int dim, double tau_active, double rho_update,
                      double delta_new, int device, dg_cluster** out);
/* Distance of the embeddings to the centroids: the `metric` argument of the reference class (clustering.py:31-46), handed to
 * scipy's cdist at mapping.py:175.  0 cosine (default), 1 euclidean, 2 sqeuclidean, 3 cityblock, 4 chebyshev; float64. */
int dg_cluster_set_metric(dg_cluster* h, int metric);
/* Processes the B chunks in order (the reference's sequential loop, diarization.py:193-203).
 * map_dev  int32 [B,K]: global speaker of each local speaker, -1 if unmapped.
 * permuted_dev float32 [B,F,M] or NULL: SpeakerMap.apply output (values are float32-exact). */
int dg_cluster_step(dg_cluster* h, const float* seg_dev /*[B,F,K]*/, const float* emb_dev /*[B,K,D]*/,
                    int B, int F, int K, int32_t* map_dev, float* permuted_dev, void* stream);
int dg_cluster_reset(dg_cluster* h);
/* synchronous host copies of the state: centers [M,D] float64, active [M] int32 (0/1);
 * *initialized = 0 until the first chunk was seen (reference `centers is None`). */
int dg_cluster_get_state(dg_cluster* h, double* centers_host, int32_t* active_host, int* initialized);
int dg_cluster_set_state(dg_cluster* h, const double* centers_host, const int32_t* active_host, int initialized);
int dg_cluster_destroy(dg_cluster* h);

/* ---- fused pipeline step: SpeakerDiarization.__call__ lines 177-203
 *      (reference src/diart/blocks/diarization.py): segmentation -> OSP -> embedding ->
 *      normalisation -> clustering, no host round trips.  The pipeline borrows the three handles. ---- */
int dg_pipeline_create(dg_seg* seg, dg_emb* emb, dg_cluster* clu, float gamma, float beta,
                       int normalize_weights, dg_pipeline** out);
int dg_pipeline_step(dg_pipeline* h, const float* wav_dev /*[B,S]*/, int B, int S,
                     float* seg_dev /*[B,F,K]*/, float* emb_dev /*[B,K,D]*/,
                     int32_t* map_dev /*[B,K]*/, float* permuted_dev /*[B,F,M] or NULL*/, void* stream);
/* Hint: consecutive windows of a batch are `hop_samples` apart in ONE stream (reference config.step x sample_rate;
 * windows as `rearrange_audio_stream` emits them, src/diart/operators.py:44-100).  The pipeline then verifies the overlap on the device for every batch (bit comparison) and, when it holds, runs the
 * sinc layer once over the unique samples instead of once per window.  0 = no hint
 * (default).  Results never depend on the hint being right. */
int dg_pipeline_set_hop(dg_pipeline* h, int hop_samples);
/* Same with HOST buffers: H2D of the waveforms and D2H of the results inside the call
 * (pinned staging owned by the handle); synchronous. */
int dg_pipeline_step_host(dg_pipeline* h, const float* wav_host, int B, int S, float* seg_host,
                          float* emb_host, int32_t* map_host, float* permuted_host /*nullable*/);
/* Pipelined variants for throughput: submit enqueues a step and returns; the sequential clustering of step i and
 * the host<->device copies overlap the networks of step i+1 (chunk order per stream is kept: all clustering runs on
 * one internal stream).  At most THREE steps may be outstanding -- two compute concurrently, the third lets the
 * waveforms of step i+2 be uploaded meanwhile -- and collect returns them oldest first.  dg_pipeline_collect makes
 * `stream` wait for the step and hands out device pointers that stay valid until the third next submit;
 * dg_pipeline_collect_host copies to host buffers and blocks. */
int dg_pipeline_submit(dg_pipeline* h, const float* wav_dev /*[B,S], must stay valid until collected*/, int B, int S,
                       void* stream);
int dg_pipeline_collect(dg_pipeline* h, const float** seg_dev, const float** emb_dev, const int32_t** map_dev,
                        void* stream);
/* as dg_pipeline_collect, but copies the step's results into caller-owned device buffers on `stream` */
int dg_pipeline_collect_copy(dg_pipeline* h, float* seg_dev, float* emb_dev, int32_t* map_dev, void* stream);
int dg_pipeline_submit_host(dg_pipeline* h, const float* wav_host /*pinned memory recommended*/, int B, int S);
int dg_pipeline_collect_host(dg_pipeline* h, float* seg_host, float* emb_host, int32_t* map_host);
/* The networks of one batch without clustering, for num_sets (1..64) overlap-aware weightings ("OSP sets"): osp_host float32
 * [num_sets][2] = {gamma, beta} (finite), normalize_host int32 [num_sets] (0 or 1).  The segmentation, the sinc front end and
 * the embedding trunk run once; the OSP weights, the pooling row weights, TDNN5 + pooling (or the un-fused pooling of the
 * WeSpeaker embedding), the finaliser and the projection run per set.  seg_dev [B,F,K]; set g's embeddings [B,K,D] at
 * emb_dev + g * emb_set_stride floats (emb_set_stride >= B K D when num_sets > 1).  Set g's outputs are the bits a pipeline
 * created with that set's gamma, beta and normalize gives in dg_pipeline_submit.  Consecutive calls alternate the two scratch
 * lanes like submitted steps, so two batches can be in flight; `stream` waits for the call's outputs, and wav_dev must stay
 * valid until then.  The sinc front end follows the hop hint (dg_pipeline_set_hop).  DG_EINVAL, with nothing launched, for bad
 * arguments or while submitted steps are outstanding. */
int dg_pipeline_nets_sets(dg_pipeline* h, const float* wav_dev, int B, int S, int num_sets, const float* osp_host,
                          const int32_t* normalize_host, float* seg_dev, float* emb_dev, int64_t emb_set_stride, void* stream);
int dg_pipeline_destroy(dg_pipeline* h);

/* ---- post-path of SpeakerDiarization.__call__ on the device (reference src/diart/blocks/diarization.py:205-232):
 *      SpeakerMap.apply (mapping.py:341-360) -> DelayedAggregation(step, latency, "hamming", "loose")
 *      (blocks/aggregation.py:73-92,120-218, incl. the first-buffer prepend rule :188-212) -> Binarize(tau)
 *      (blocks/utils.py:11-59), run-length encoded.  The handle keeps the scores / maps of the last num_windows - 1
 *      chunks (the reference's pred_buffer) on the device; num_windows = round(latency / step).
 *      hamming_host = np.hamming(frames) in float64.  Arithmetic is float64 in numpy's order without fused
 *      multiply-add: the thresholded result is bit-identical to the reference's.
 *
 *      plan_host int32 [B][4 + num_windows], one row per chunk, computed by the host with pyannote.core's
 *      SlidingWindow.crop index arithmetic (diart_b200/blocks/post.py):
 *        [0] nb   buffers aggregated for this chunk (1 .. num_windows)
 *        [1] nf   frames of the aggregated region
 *        [2] first_nf  > 0 only for the first buffer of a stream: output = first_nf frames, the last nf aggregated
 *        [3] first_lo  first frame of that prepended crop (may be negative: edge-padded)
 *        [4 + j]  first frame of buffer j's crop (oldest buffer first; may leave [0, frames): edge-padded)
 *      header_host int32 [B][4] = {offset into turns, number of turns, output frames, 0};
 *      turns_host  uint32 [turn_cap_host], packed speaker << 20 | on << 10 | off (frame indices; the turn covers the
 *      frame MIDDLES on .. off as in Binarize), each chunk's turns contiguous, by speaker then time.
 *      dg_post_step synchronises `stream`. ---- */
int dg_post_create(int frames, int local_speakers, int max_speakers, int num_windows, const double* hamming_host,
                   double tau, int device, dg_post** out);
int dg_post_step(dg_post* h, const float* seg_dev /*[B,F,K]*/, const int32_t* map_dev /*[B,K]*/, int B,
                 const int32_t* plan_host, int32_t* header_host, uint32_t* turns_host, int turn_cap_host, int* n_turns,
                 void* stream);
int dg_post_reset(dg_post* h);
int dg_post_destroy(dg_post* h);
/* The whole body of SpeakerDiarization.__call__ (reference diarization.py:172-232) in ONE call: rows_host[b] points to the
 * S float32 samples of window b (B separate host arrays, as rearrange_audio_stream emits them).  With a hop set
 * (dg_pipeline_set_hop) worker threads compare every window with its predecessor (memcmp of the S - hop shared samples);
 * windows that are consecutive hops of one stream are uploaded ONCE (S + (B-1) hop samples) and formed on the device,
 * anything else is gathered into pinned staging and uploaded as [B,S] while the gather is still running.  Then fused step
 * + post-path in up to three pipelined sub-batches; only the turn list (and, if asked for, scores and maps) returns to
 * the host.  Synchronous.  dg_pipeline_last_call_h2d_bytes: what the last call uploaded. */
int dg_pipeline_call_host(dg_pipeline* h, dg_post* post, const float* const* rows_host, int B, int S,
                          const int32_t* plan_host, int32_t* header_host, uint32_t* turns_host, int turn_cap_host,
                          int* n_turns, float* seg_host /*nullable*/, int32_t* map_host /*nullable*/);
int64_t dg_pipeline_last_call_h2d_bytes(const dg_pipeline* h);

/* ---- hyper-parameter sweep: the reference tunes tau_active, rho_update and delta_new by running its whole pipeline once per
 *      trial over every file (Optimizer.objective -> Benchmark, reference src/diart/optim.py:98-122, inference.py:392-432).
 *      None of the three reaches the networks, so here one file's network outputs (seg_dev [N,F,K], emb_dev [N,K,D], e.g.
 *      from dg_pipeline_submit / collect) are clustered and post-processed for T trials at once: T independent
 *      OnlineSpeakerClustering states (cosine, max_speakers), each followed by the dg_post_* post-path with its own tau, all
 *      N chunks in one pass without history.  Per trial the result is the one a fresh pipeline with that trial's thresholds
 *      produces over the same N chunks.
 *      dg_sweep_create takes the limits of dg_cluster_create and dg_post_create (max_speakers <= 32, local_speakers <= 8 and
 *      <= max_speakers, frames <= 1023, 1 <= num_windows <= 256) and hamming_host = np.hamming(frames) in float64.
 *      dg_sweep_run:
 *        params_host float64 [T][3] = {tau_active, rho_update, delta_new} per trial (finite), 1 <= T <= 65535, N >= 1;
 *        plan_host   int32 [N][4 + num_windows]: the dg_post_step plan of the N chunks as ONE batch of a fresh stream;
 *        maps_dev    int32 [T][N][K] or NULL: each trial's speaker maps (dg_cluster_step's map_dev);
 *        centers_dev float64 [T][M][D] or NULL: each trial's final centroids (zero rows for inactive speakers);
 *        header_host int32 [T][N][4] and turns_host uint32 [turn_cap_host]: as dg_post_step, the turns of all trials in one
 *        list, located by each trial's headers.  When the turns exceed turn_cap_host the call fails with DG_EINVAL and
 *        *n_turns holds the count needed.
 *      Synchronous (synchronises `stream`). ---- */
int dg_sweep_create(int max_speakers, int dim, int frames, int local_speakers, int num_windows, const double* hamming_host,
                    int device, dg_sweep** out);
int dg_sweep_run(dg_sweep* h, const float* seg_dev, const float* emb_dev, int N, const double* params_host, int T,
                 const int32_t* plan_host, int32_t* maps_dev, double* centers_dev, int32_t* header_host, uint32_t* turns_host,
                 int turn_cap_host, int* n_turns, void* stream);
int dg_sweep_destroy(dg_sweep* h);
/* ---- dg_sweep_set_scored_regions / dg_vad_sweep_set_scored_regions: the scored regions of a metric with a forgiveness
 *      collar, skip_overlap or a uem (DESIGN.md "DER scoring", steps 1-4) for the handle's later scoring calls.  File f's
 *      pieces are rows_host float64 [S][2] {start, end} at [offsets_host[f], offsets_host[f + 1]) (int32 [num_files + 1] from
 *      0, not decreasing): sorted, each more than 1e-6 s long and starting more than 1e-6 s after the previous one ends, all
 *      finite; otherwise DG_EINVAL and the previous regions stay.  Every (file, trial) hypothesis is cropped to its file's
 *      pieces before the scoring walk; the caller passes references already cropped to them.  num_files = 0 clears them (the
 *      default: hypotheses scored whole).  While they are set, every dg_sweep_score* / dg_vad_sweep_score_files call must
 *      score exactly num_files files (the virtual files of the _latencies entry points and of a curve over several
 *      latencies), else DG_EINVAL before any launch.  Host only (the pieces travel with the next scoring call). ---- */
int dg_sweep_set_scored_regions(dg_sweep* h, int num_files, const double* rows_host, const int32_t* offsets_host);
int dg_vad_sweep_set_scored_regions(dg_vad_sweep* h, int num_files, const double* rows_host, const int32_t* offsets_host);
/* ---- dg_sweep_set_trial_sets: sweeps over overlap-aware weightings (dg_pipeline_nets_sets).  For the handle's later
 *      dg_sweep_run* / dg_sweep_score* calls emb_dev is [num_sets][N][K][D] (the embeddings of every set over the same
 *      chunks), and trial t's clustering reads set trial_set_host[t] (int32 [T], each in [0, num_sets)); the post-path and the
 *      scoring read only the scores and maps and are unchanged.  Every such call must run exactly T trials, else DG_EINVAL
 *      before any launch.  num_sets = 0 clears them (the default: emb_dev is [N][K][D]).  DG_EINVAL for an index out of range
 *      or num_sets outside 0..64, and the previous state stays.  Host only. ---- */
int dg_sweep_set_trial_sets(dg_sweep* h, int num_sets, const int32_t* trial_set_host, int T);
/* ---- dg_sweep_set_seeds: known speakers for the handle's later dg_sweep_run* / dg_sweep_score* calls.  File f's known
 *      centroids are rows [offsets_host[f], offsets_host[f + 1]) of centers_host float64 [n][D] (offsets int32 [num_files + 1]
 *      from 0, not decreasing).  The files are the ones a call clusters: one for dg_sweep_run / dg_sweep_score, the files of
 *      the _files entry points, the units of the _latencies ones.  Every (file, trial) state then starts as
 *      dg_multi_open_seeded starts a stream: centres 0 .. n_f - 1 hold the centroids and are active, and the state counts as
 *      initialised when n_f > 0 (so the clustering takes the distance path from the first chunk); a file without centroids
 *      starts fresh.  num_files = 0 clears them (the default).  DG_EINVAL, changing nothing, for offsets that do not start at 0
 *      or decrease, more than max_speakers centroids for one file, or a centroid that is not finite or has a zero norm.  A
 *      later call that clusters another number of files gets DG_EINVAL before any launch.  Host only (the centroids travel in
 *      the next call's upload). ---- */
int dg_sweep_set_seeds(dg_sweep* h, int num_files, const int32_t* offsets_host, const double* centers_host);
/* ---- dg_sweep_set_identities: identification error (DESIGN.md "Identification error") for the handle's later
 *      dg_sweep_score* calls.  hyp_of_ref_host int32 [num_files][32]: for each scored file (the virtual files of
 *      dg_sweep_score_latencies) and reference label r (string order, as the reference rows number them), the hypothesis label
 *      g of the same name, or -1.  Each reference label is then matched to that label instead of by the optimal mapping; the
 *      five components are otherwise computed as for DER.  Entries for r >= the file's label count are ignored.  num_files = 0
 *      clears the table (the default: DER).  DG_EINVAL, changing nothing, for an entry outside [-1, max_speakers) or a g given
 *      twice in one file.  A later scoring call over another number of files gets DG_EINVAL before any launch.  Host
 *      only. ---- */
int dg_sweep_set_identities(dg_sweep* h, int num_files, const int32_t* hyp_of_ref_host);
/* ---- dg_sweep_score: the same clustering and post-path as dg_sweep_run, then each trial's diarization error rate components
 *      against one reference (DiarizationErrorRate, the metric of the reference's Benchmark.evaluate; definition in
 *      DESIGN.md "DER scoring"): collar=0, skip_overlap=False and no uem, or, with scored regions set
 *      (dg_sweep_set_scored_regions), the hypothesis cropped to them and the reference as given (cropped by the caller).
 *      The turns never leave the device.
 *        seg_dev ... plan_host   as dg_sweep_run;
 *        out_start_host, out_res_host float64 [N]: each chunk's output start and frame resolution (blocks/post.py post_plan),
 *        shift: added to every turn time (the file's timestamp shift), collar >= 0: the merge collar of the whole-file
 *        prediction (PredictionAccumulator's, 0.05 s);
 *        ref_host float64 [S][2] {start, end} with start < end, ref_label_host int32 [S] in [0, R), R <= 32 labels; the rows of
 *        one label in time order and not overlapping (touching is allowed);
 *        components_host float64 [T][5] = {false alarm, missed detection, confusion, correct, total} seconds;
 *        hyp_offsets_dev int32 [T * max_speakers + 1] or NULL: offsets of each (trial, label)'s merged hypothesis segments,
 *        hyp_segments_dev float64 [hyp_cap][2] or NULL: the segments {start, end}, (trial, label) major, in time order.  When
 *        they exceed hyp_cap the call fails with DG_EINVAL after writing the components and the offsets.
 *      Every argument is checked before any launch.  Synchronous (synchronises `stream`). ---- */
int dg_sweep_score(dg_sweep* h, const float* seg_dev, const float* emb_dev, int N, const double* params_host, int T,
                   const int32_t* plan_host, const double* out_start_host, const double* out_res_host, double shift,
                   double collar, const double* ref_host, const int32_t* ref_label_host, int S, int R,
                   double* components_host, int32_t* hyp_offsets_dev, double* hyp_segments_dev, int hyp_cap, void* stream);
/* ---- dg_sweep_run_files / dg_sweep_score_files: the same for a dataset of num_files files in ONE launch per kernel (the
 *      reference's Optimizer.objective scores a trial over every file of a dataset).  seg_dev / emb_dev hold the files'
 *      chunks concatenated, N in all; file f owns chunks [chunk_offsets_host[f], chunk_offsets_host[f + 1]), with
 *      chunk_offsets_host int32 [num_files + 1] starting at 0, ending at N and increasing (every file has a chunk).  A state is
 *      a (file, trial) pair: a fresh clustering per file and trial, exactly what dg_sweep_run / dg_sweep_score give for that
 *      file alone; num_files * T <= 2^21.  The clustering CTAs run longest file first (dg_sweep_state_order); the order
 *      changes no result.
 *        plan_host, out_start_host, out_res_host: each file's own (a fresh stream per file), concatenated;
 *        maps_dev int32 [T][N][K], header_host int32 [T][N][4]: as dg_sweep_run over the concatenated chunks;
 *        centers_dev float64 [num_files][T][M][D];
 *        shifts_host float64 [num_files]: each file's timestamp shift;
 *        ref_host [S][2] / ref_label_host [S]: the files' reference rows concatenated, file f's at rows
 *        [ref_offsets_host[f], ref_offsets_host[f + 1]) (int32 [num_files + 1] from 0, not decreasing) with labels in
 *        [0, ref_label_counts_host[f]) (int32 [num_files], each <= 32), checked per file as dg_sweep_score's;
 *        components_host float64 [num_files][T][5];
 *        hyp_offsets_dev int32 [num_files * T * max_speakers + 1] or NULL: (file, trial, label) major.
 *      Every argument is checked before any launch.  Synchronous (synchronises `stream`). ---- */
int dg_sweep_run_files(dg_sweep* h, const float* seg_dev, const float* emb_dev, int N, int num_files,
                       const int32_t* chunk_offsets_host, const double* params_host, int T, const int32_t* plan_host,
                       int32_t* maps_dev, double* centers_dev, int32_t* header_host, uint32_t* turns_host, int turn_cap_host,
                       int* n_turns, void* stream);
int dg_sweep_score_files(dg_sweep* h, const float* seg_dev, const float* emb_dev, int N, int num_files,
                         const int32_t* chunk_offsets_host, const double* params_host, int T, const int32_t* plan_host,
                         const double* out_start_host, const double* out_res_host, const double* shifts_host, double collar,
                         const double* ref_host, const int32_t* ref_label_host, const int32_t* ref_offsets_host,
                         const int32_t* ref_label_counts_host, double* components_host, int32_t* hyp_offsets_dev,
                         double* hyp_segments_dev, int hyp_cap, void* stream);
/* the launch order of the (file, trial) states of dg_sweep_*_files, states_host int32 [num_files * T][2] = {file, trial}:
 * longest file first (equal chunk counts in file order), then trial.  Host only. */
int dg_sweep_state_order(int num_files, const int32_t* chunk_offsets_host, int T, int32_t* states_host);
/* ---- dg_sweep_run_latencies / dg_sweep_score_latencies: dg_sweep_*_files at several latencies from one set of network
 *      outputs.  A file's windows at a smaller latency are a prefix of its windows at a larger one with the same left
 *      padding.  seg_dev / emb_dev hold the chunks of num_units *units*, N in all, unit u at [unit_offsets_host[u],
 *      unit_offsets_host[u + 1]) (as chunk_offsets_host above); a unit is the windows of one file at the largest latency of a
 *      group whose outputs are prefixes of the unit's, bit for bit (the caller groups them).  A *virtual file* is one
 *      (latency, file) pair, the first chunks of its unit; the num_virtual_files virtual files hold the num_virtual virtual
 *      chunks, virtual file v at [virtual_offsets_host[v], virtual_offsets_host[v + 1]) (int32 [num_virtual_files + 1] from 0
 *      to num_virtual, increasing), and vchunk_host int32 [num_virtual] gives the real chunk of each virtual chunk.  Every
 *      virtual file must be the real chunks u0, u0 + 1, ... of one unit starting at its first chunk u0 and not crossing into
 *      the next unit, and every plan row must aggregate no buffer before that first chunk, at most num_windows (the
 *      handle's) of them, over at most frames + 1 output frames; otherwise DG_EINVAL before any launch.
 *        params_host float64 [T][3] as dg_sweep_run: the clustering runs once per (unit, trial) for the units some virtual
 *        file starts at, longest unit first, whatever the number of latencies;
 *        plan_host int32 [num_virtual][4 + num_windows]: each virtual file's plan at its own latency (a fresh stream),
 *        zero-padded to the handle's num_windows (that of the largest latency);
 *        maps_dev int32 [T][N][K] or NULL: over the real chunks (those of units no virtual file reads are not written);
 *        header_host int32 [T][num_virtual][4], turns: as dg_sweep_run_files over the virtual chunks;
 *        out_start_host, out_res_host float64 [num_virtual], shifts_host float64 [num_virtual_files] and the references
 *        (ref_offsets_host, ref_label_counts_host per virtual file) as dg_sweep_score_files with the virtual files as files;
 *        components_host float64 [num_virtual_files][T][5]; num_virtual_files * T <= 2^21.
 *      For a virtual file of latency L every result is what dg_sweep_*_files gives for that file's windows at latency L
 *      alone.  One difference: a clustering error ("Cannot update unknown centers") in the chunks of a unit beyond a smaller
 *      latency's prefix fails the call for every latency that reads the unit, not only for those whose windows reach it.
 *      Synchronous.
 *      dg_sweep_check_latencies: the layout checks alone, for a handle of num_windows and frames (host only, no device). ---- */
int dg_sweep_run_latencies(dg_sweep* h, const float* seg_dev, const float* emb_dev, int N, int num_units,
                           const int32_t* unit_offsets_host, int num_virtual, int num_virtual_files, const int32_t* vchunk_host,
                           const int32_t* virtual_offsets_host, const double* params_host, int T, const int32_t* plan_host,
                           int32_t* maps_dev, int32_t* header_host, uint32_t* turns_host, int turn_cap_host, int* n_turns,
                           void* stream);
int dg_sweep_score_latencies(dg_sweep* h, const float* seg_dev, const float* emb_dev, int N, int num_units,
                             const int32_t* unit_offsets_host, int num_virtual, int num_virtual_files,
                             const int32_t* vchunk_host, const int32_t* virtual_offsets_host, const double* params_host, int T,
                             const int32_t* plan_host, const double* out_start_host, const double* out_res_host,
                             const double* shifts_host, double collar, const double* ref_host, const int32_t* ref_label_host,
                             const int32_t* ref_offsets_host, const int32_t* ref_label_counts_host, double* components_host,
                             void* stream);
int dg_sweep_check_latencies(int N, int num_units, const int32_t* unit_offsets_host, int num_virtual, int num_virtual_files,
                             const int32_t* vchunk_host, const int32_t* virtual_offsets_host, const int32_t* plan_host,
                             int num_windows, int frames);
/* ---- voice activity detection sweep: the reference tunes VoiceActivityDetection's one hyper-parameter, tau_active, by
 *      running the whole pipeline per trial and file and scoring it with DetectionErrorRate(collar=0, skip_overlap=False)
 *      (reference blocks/vad.py:108-114, optim.py:98-122); with scored regions set (dg_vad_sweep_set_scored_regions) any
 *      collar, skip_overlap and uem.  tau_active is read by Binarize alone, so here the speech curve of
 *      every chunk (max over the local speakers, Hamming-aggregated as dg_post_step with one speaker) is computed once per
 *      dataset and kept on the device; each trial thresholds it.
 *      dg_vad_sweep_create: frames <= 1023, 1 <= local_speakers <= 64, 1 <= num_windows <= 256, hamming_host =
 *      np.hamming(frames) in float64.
 *      dg_vad_sweep_curve: seg_dev float32 [N][frames][local_speakers], the segmentation scores of num_files files'
 *        chunks concatenated, file f's at [chunk_offsets_host[f], chunk_offsets_host[f + 1]) (int32 [num_files + 1] from 0 to
 *        N, increasing); plan_host int32 [N][4 + num_windows]: each file's dg_post_step plan as one batch of a fresh stream,
 *        concatenated.  Computes and keeps the curve (one float64 per output frame; seg_dev is no longer read afterwards).
 *        Synchronous.
 *      dg_vad_sweep_run_files: taus_host float64 [T] (finite), 1 <= T <= 65535, num_files * T <= 2^21; header_host int32
 *        [T][N][4] and turns_host as dg_sweep_run_files (one speaker, 0).  Synchronous.
 *      dg_vad_sweep_score_files: out_start_host, out_res_host float64 [N], shifts_host float64 [num_files] and collar as
 *        dg_sweep_score_files; ref_host float64 [S][2]: each file's speech reference as one label, the support of all its
 *        segments (cropped to the file's scored regions when they are set; rows in time order, each more than 1e-6 s after the previous one), file f's at rows
 *        [ref_offsets_host[f], ref_offsets_host[f + 1]) (int32 [num_files + 1] from 0, not decreasing);
 *        components_host float64 [num_files][T][2] = {false alarm, missed detection} seconds.  The total (the reference's
 *        duration) does not depend on the trial and is the caller's.  Synchronous.
 *      dg_vad_sweep_curve_latencies: the curve over the virtual layout of several latencies (units, virtual chunks and files,
 *        plan zero-padded to the handle's num_windows, all as dg_sweep_run_latencies): virtual chunk c's curve is that of
 *        real chunk vchunk_host[c] at its virtual file's latency.  Afterwards the handle's N and files are the virtual chunks
 *        and files: dg_vad_sweep_run_files / dg_vad_sweep_score_files threshold and score every (latency, file) pair, with
 *        out_start, out_res, shifts and references per virtual chunk and file.  Synchronous.
 *      Every argument is checked before any launch. ---- */
int dg_vad_sweep_create(int frames, int local_speakers, int num_windows, const double* hamming_host, int device,
                        dg_vad_sweep** out);
int dg_vad_sweep_curve(dg_vad_sweep* h, const float* seg_dev, int N, int num_files, const int32_t* chunk_offsets_host,
                       const int32_t* plan_host, void* stream);
int dg_vad_sweep_curve_latencies(dg_vad_sweep* h, const float* seg_dev, int N, int num_units, const int32_t* unit_offsets_host,
                                 int num_virtual, int num_virtual_files, const int32_t* vchunk_host,
                                 const int32_t* virtual_offsets_host, const int32_t* plan_host, void* stream);
int dg_vad_sweep_run_files(dg_vad_sweep* h, const double* taus_host, int T, int32_t* header_host, uint32_t* turns_host,
                           int turn_cap_host, int* n_turns, void* stream);
int dg_vad_sweep_score_files(dg_vad_sweep* h, const double* taus_host, int T, const double* out_start_host,
                             const double* out_res_host, const double* shifts_host, double collar, const double* ref_host,
                             const int32_t* ref_offsets_host, double* components_host, void* stream);
int dg_vad_sweep_destroy(dg_vad_sweep* h);

/* ---- device-side audio stream: rearrange_audio_stream (reference src/diart/operators.py:44-100) with the ring buffer in
 *      HBM.  The host pushes every sample ONCE (step_samples new samples per chunk instead of chunk_samples: 8.2 MB
 *      instead of 82 MB per 256-chunk step at 5 s / 0.5 s); window i of the stream is samples
 *      [i * step_samples, i * step_samples + chunk_samples).  max_windows = largest batch that will be requested.
 *      dg_stream_push_host may be called with any block size (the reference's sources emit arbitrary blocks); it
 *      fails with DG_EINVAL when the ring is full, i.e. windows must be consumed first. ---- */
int dg_stream_create(int chunk_samples, int step_samples, int max_windows, int device, dg_stream** out);
int dg_stream_push_host(dg_stream* h, const float* samples_host, int n);
/* complete windows pushed but not yet consumed */
int dg_stream_available(const dg_stream* h);
/* the next B windows as a dense [B, chunk_samples] device batch on `stream`; advances the stream by B steps */
int dg_stream_windows(dg_stream* h, int B, float* wav_dev, void* stream);
int dg_stream_reset(dg_stream* h);
int dg_stream_destroy(dg_stream* h);
/* dg_pipeline_submit_host / dg_pipeline_call_host whose batch is the next B windows of `stream` (no window upload; the
 * sinc layer takes its stream form directly: the windows overlap by construction).  Collect with dg_pipeline_collect*. */
int dg_pipeline_submit_stream(dg_pipeline* h, dg_stream* stream, int B);
int dg_pipeline_call_stream(dg_pipeline* h, dg_post* post, dg_stream* stream, int B, const int32_t* plan_host,
                            int32_t* header_host, uint32_t* turns_host, int turn_cap_host, int* n_turns,
                            float* seg_host /*nullable*/, int32_t* map_host /*nullable*/);

/* ---- many live streams on one device: the reference's live loop (src/diart/inference.py: StreamingInference with
 *      batch_size=1, one window per stream every step) runs SpeakerDiarization.__call__ (src/diart/blocks/diarization.py:172-232)
 *      once per stream and window.  A dg_multi owns up to max_streams such streams, all with one configuration and the same
 *      model handles, and serves them in ticks: every open stream gives its complete, unconsumed windows (at most
 *      max_windows_per_stream) and they run as ONE batch, with every stream's result that of its own pipeline.
 *      dg_multi_create: chunk_samples / step_samples positive multiples of 4 (window i of a stream is samples
 *        [i * step, i * step + chunk)); max_streams * max_windows_per_stream <= 65535; tau, rho, delta = tau_active,
 *        rho_update, delta_new (cosine clustering with max_speakers <= 32 centres; tau_active also binarises); gamma, beta,
 *        normalize_weights as dg_pipeline_create; num_windows = max_latency / step, the largest number of aggregated
 *        buffers of any stream (sizes every slot's history), and hamming_host = np.hamming(frames) in float64, as
 *        dg_post_create.  tau, rho, delta and num_windows are also the values of a stream opened without its own.  The model
 *        handles are borrowed and may serve other pipelines meanwhile.
 *      dg_multi_open: a new stream in `slot` (0 <= slot < max_streams, not open) at the handle's values: no samples, fresh
 *        clustering state (the reference's reset()), no aggregation history.  dg_multi_close: the stream in `slot` ends; its
 *        staged samples are dropped.
 *      dg_multi_open_config: dg_multi_open_rate with the stream's own latency and thresholds, fixed until it is closed:
 *        num_windows = its latency / step (1 <= num_windows <= the handle's num_windows) buffers aggregated, params = {tau,
 *        rho, delta} (tau_active, rho_update, delta_new; a VAD handle reads params[0] only).  Its results are those of a
 *        dedicated pipeline at those values; its plan rows (dg_multi_step) are plan rows of that latency.  DG_EINVAL, naming
 *        dg_multi_open_config and changing nothing, unless the slot and rate are as dg_multi_open_rate needs, num_windows is
 *        in range and the values read are finite.
 *      dg_multi_push_host: appends n samples (any block size) to the stream in `slot`.  They are copied to pinned staging;
 *        nothing reaches the device before the next tick.  Fails with DG_EINVAL, writing nothing, if the stream would hold
 *        more unconsumed samples than its ring (chunk + 2 max_windows_per_stream step, rounded up to 1024).
 *      dg_multi_available: complete windows of the stream in `slot` not yet consumed (staged samples included), or DG_EINVAL.
 *      dg_multi_step: one tick.  Every open slot s, in slot order, gives n_s = min(available, max_windows_per_stream) windows;
 *        counts_host int32 [max_streams] receives n_s.  The n_rows = sum n_s chunks are the tick's rows, grouped by slot, each
 *        slot's in window order; plan_host int32 [n_rows][4 + num_windows] holds their dg_post_step plan rows at each
 *        stream's own latency (a chunk's row depends only on its window index within its stream and that latency:
 *        diart_b200.serve.plan_rows), a row of a stream with fewer buffers leaving the tail unused.  n_rows must equal sum
 *        n_s and no row may aggregate more buffers than its stream's num_windows, else DG_EINVAL.  header_host int32 [n_rows][4] and turns_host as dg_post_step.  seg_dev [n_rows, F, K], emb_dev
 *        [n_rows, K, D] and map_dev [n_rows, K] (device, nullable) receive the tick's network outputs and speaker maps.  All
 *        staged samples go up in one copy; the networks run in sub-batches of at most 256 windows.  A tick without windows
 *        launches nothing.  Every argument is checked before any launch.  Synchronous. ---- */
typedef struct dg_multi dg_multi;
int dg_multi_create(dg_seg* seg, dg_emb* emb, int chunk_samples, int step_samples, int max_streams, int max_windows_per_stream,
                    int max_speakers, double tau, double rho, double delta, float gamma, float beta, int normalize_weights,
                    int num_windows, const double* hamming_host, dg_multi** out);
int dg_multi_open(dg_multi* h, int slot);
int dg_multi_close(dg_multi* h, int slot);
int dg_multi_push_host(dg_multi* h, int slot, const float* samples_host, int n);
int dg_multi_available(const dg_multi* h, int slot);
int dg_multi_step(dg_multi* h, const int32_t* plan_host, int n_rows, int32_t* counts_host, int32_t* header_host,
                  uint32_t* turns_host, int turn_cap_host, int* n_turns, float* seg_dev /*nullable*/,
                  float* emb_dev /*nullable*/, int32_t* map_dev /*nullable*/);
/* device time of the last tick that had windows, from events on the handle's stream around all of its device work (upload,
 * networks, clustering, post-path, download), in ms; DG_EINVAL before the first such tick */
int dg_multi_last_step_ms(const dg_multi* h, float* ms);
int dg_multi_destroy(dg_multi* h);
/* ---- streams at other source rates (a microphone at 44.1 kHz, say), resampled on the device as the reference's
 *      blocks.Resample resamples every window (src/diart/inference.py:101-123).
 *      dg_multi_add_rate: declares the source rate of `rs` (borrowed, on the handle's device; dg_resample_create(rate,
 *        pipeline rate)) with chunk_samples / step_samples source samples per window / between windows (window i of such a
 *        stream is source samples [i * step, i * step + chunk), resampled).  *rate_id receives 0, 1, ... in declaration
 *        order.  Only before the first dg_multi_open*, because it grows the rings.  DG_EINVAL, changing nothing, unless the
 *        chunk resamples to exactly the handle's chunk_samples, step % o == 0 (o / n the reduced rate ratio: a hop is whole
 *        output frames), step <= chunk, the rate was not declared before and its rings fit 2^30 samples per stream.
 *        Memory: every slot's source ring grows to the largest capacity (chunk + 2 max_windows_per_stream step, rounded up to
 *        1024) of any rate, and every slot gets a 16 kHz ring of ((max_windows_per_stream - 1) step / o + r_hi - r_lo + 1) n
 *        floats (the interior frames of max_windows_per_stream consecutive windows), largest over the rates.
 *      dg_multi_open_rate: dg_multi_open at declared rate `rate_id` (-1: the pipeline's rate, = dg_multi_open).
 *        dg_multi_push_host and dg_multi_available then count source samples and source-rate windows, and the capacity of
 *        the slot is its rate's: a stream at the pipeline's rate refuses exactly what it refuses without declared rates.
 *      In a tick, a resampled stream's windows are computed from its source ring: each 16 kHz frame whose taps all lie inside
 *        a window is computed once over the life of the stream (one launch per rate in the tick, kept in the slot's 16 kHz
 *        ring), and the frames at each window's edges are recomputed with the window's zero padding.  Every resampled window
 *        has the bits of dg_resample_forward on the stacked source window.  A tick whose streams are all at the pipeline's
 *        rate launches what it launches without declared rates. ---- */
typedef struct dg_resample dg_resample;   /* declared with its entry points below */
int dg_multi_add_rate(dg_multi* h, dg_resample* rs, int chunk_samples, int step_samples, int* rate_id);
int dg_multi_open_rate(dg_multi* h, int slot, int rate_id);
int dg_multi_open_config(dg_multi* h, int slot, int rate_id, int num_windows, const double params[3] /* tau, rho, delta */);
/* ---- known speakers: a stream that starts from a given clustering state (diart_b200.speakers).  The reference's
 *      OnlineSpeakerClustering.identify (src/diart/blocks/clustering.py:149) takes its first-chunk path only while its centers
 *      are None; a state filled beforehand goes straight to the distance path.
 *      dg_multi_open_seeded: dg_multi_open_config, with the slot's clustering state seeded from centers_host float64 [n][D]:
 *        rows 0 .. n - 1 written from it and active, rows n .. max_speakers - 1 zero, initialised iff n > 0 (n = 0 is
 *        dg_multi_open_config).  The writes are ordered on the handle's stream; centers_host may be freed when the call
 *        returns.  DG_EINVAL, naming dg_multi_open_seeded and changing nothing, if dg_multi_open_config would refuse, the
 *        handle is a VAD handle, n < 0 or n > max_speakers, or a centroid is not finite or has a zero norm.
 *      dg_multi_get_state: the clustering state of the open stream in `slot` after its last tick: centers_host float64
 *        [max_speakers][D], active_host int32 [max_speakers] (1: active), *initialized.  DG_EINVAL for a closed slot or a VAD
 *        handle.  Synchronous (dg_multi_step is, so the state is that of the last tick). ---- */
int dg_multi_open_seeded(dg_multi* h, int slot, int rate_id, int num_windows, const double params[3] /* tau, rho, delta */,
                         const double* centers_host /* [n][D] */, int n);
int dg_multi_get_state(dg_multi* h, int slot, double* centers_host /* [M][D] */, int32_t* active_host /* [M] */,
                       int* initialized);
/* ---- speaker gallery: names for discovered speakers from an enrolled gallery of any size (DESIGN.md "Gallery naming").
 *      The cosine distance 1 - clip(u.v / (|u| |v|), -1, 1) is evaluated in float64 (dot products on the float64 tensor
 *      cores, each summed in one fixed order: identical entries give identical distances).
 *      dg_gallery_create: uploads centroids_host float64 [G][D] to `device` and computes the entries' norms.  DG_EINVAL unless
 *        1 <= G <= 1048576, D >= 2 is even, and every entry is finite with a non-zero norm.
 *      dg_gallery_query: per query q of queries_dev float64 [Q][D] (row stride D), on `stream`: dist_dev [q] the distance to
 *        the nearest entry its group has not claimed (ties: the lowest entry; +inf when none is left), entry_dev [q] that
 *        entry if the distance is < threshold and q wins it within its group, else -1.  group_dev int32 [Q]: the query's claim
 *        group, >= 0, each group one contiguous run of at most 32 queries; claimed_dev int32 [groups][32] (null: none): the
 *        entries group r has claimed, -1 padded.  Within a group, candidates for one entry are resolved by the smallest
 *        distance, ties to the earliest query.  group_dev is read back on `stream` (the call waits for it) to check it.
 *        Queries of more than 2^31 - 1 elements are searched in several launches of whole groups (DG_EINVAL only when
 *        one group alone exceeds that: a dimension above 67 million).
 *      dg_multi_set_gallery: every later tick names the active, unnamed global speakers of its streams from the gallery
 *        (dg_multi_last_names).  DG_EINVAL on a VAD handle, once a stream has opened, for a gallery of another dimension or
 *        device, or unless 0 < threshold <= 2.
 *      dg_multi_set_slot_gallery: the stream in `slot` is named from gallery g at `threshold` instead of the default
 *        (dg_multi_set_gallery) for the rest of its life, starting with nothing named or claimed.  Any number of streams
 *        may have their own galleries, the same or different ones; a tick searches all of them in one grouped launch.  The
 *        handle refers to g until the slot is closed: g must outlive that.  DG_EINVAL for a null handle or gallery, a VAD
 *        handle, a slot that is not open or has had a tick, a gallery of another dimension or device, or unless
 *        0 < threshold <= 2.
 *      dg_multi_set_names: the names of the open stream in `slot` (a slot with a gallery, its own or the default): bit g of
 *        `named` set for a named global speaker g < max_speakers, claimed_host int32 [max_speakers] its entry in the slot's
 *        gallery (-1: none; only named speakers claim, each entry once).  A stream opens with none named.
 *      dg_multi_last_names: the names decided by the last dg_multi_step, out_host int32 [cap][3] = {slot, g, entry}, *n of
 *        them; DG_EINVAL if more than cap. ---- */
typedef struct dg_gallery dg_gallery;
int dg_gallery_create(const double* centroids_host, int G, int D, int device, dg_gallery** out);
int dg_gallery_destroy(dg_gallery* g);
int dg_gallery_query(dg_gallery* g, const double* queries_dev /* [Q][D] */, int Q, const int32_t* group_dev /* [Q] */,
                     const int32_t* claimed_dev /* [groups][32] */, double threshold, int32_t* entry_dev /* [Q] */,
                     double* dist_dev /* [Q] */, void* stream);
int dg_multi_set_gallery(dg_multi* h, dg_gallery* g, double threshold);
int dg_multi_set_slot_gallery(dg_multi* h, int slot, dg_gallery* g, double threshold);
int dg_multi_set_names(dg_multi* h, int slot, uint32_t named, const int32_t* claimed_host /* [max_speakers] */);
int dg_multi_last_names(const dg_multi* h, int32_t* out_host /* [cap][3] */, int cap, int* n);
/* test hook: the last tick's window batch [n_rows, chunk_samples] (what its networks read; n_rows = that tick's window count)
 * copied to wav_dev.  Synchronous. */
int dg_multi_last_windows(const dg_multi* h, float* wav_dev, int n_rows);
/* ---- moving live streams between handles (diarization and VAD handles alike), e.g. to drain a GPU, rebalance or keep a
 *      checkpoint.  A stream's packed state holds everything its next ticks read, so the stream continues on the target
 *      exactly as on the source.  Layout, format version 1 (host byte order; every section starts at a multiple of 16 bytes
 *      from the state's start, and a state's size is a multiple of 16, so states follow each other directly):
 *        head (a fixed struct, csrc/api_multi.cu XferHead): magic "DGST", version, kind (0 diarization, 1 VAD); the
 *          pipeline's window and step samples, F, K, D, M; the source rate's resampling {o, n, w} (all 0 at the pipeline's
 *          rate), window and step at that rate; the stream's buffers (latency / step) and history entries n_hist; the
 *          clustering's two init words; the named speakers (bit g) and the size of the gallery they are named from (0:
 *          none); whether it has had a tick; the absolute wpos, rpos and done (16 kHz frames computed), and the frames
 *          carried [frame0, frame0 + n_frames); {tau, rho, delta}; the gallery threshold; gamma, beta,
 *          normalize_weights; the state's bytes;
 *        audio float32 [wpos - rpos]: the samples from the start of the next window on, staged ones included;
 *        frames float32 [n_frames][n]: for a resampled stream, the computed 16 kHz frames a future window still reads;
 *        history, oldest first: diarization scores float32 [n_hist][F][K] then maps int32 [n_hist][K]; VAD max curves
 *          float32 [n_hist][F];
 *        diarization only: centroids float64 [M][D], active int32 [32], claimed gallery entries int32 [32] (-1: none).
 *      dg_multi_export_bytes: the size of each listed slot's state now (it grows with pushes).
 *      dg_multi_export: the states of the n listed open slots (distinct), packed in list order into out_host (out_bytes:
 *        its size).  One launch gathers the device state of every slot of a round into a staging buffer, one copy brings
 *        it back through pinned memory (rounds of at most 256 MiB of states).  close != 0 then closes the slots as
 *        dg_multi_close does; close = 0 leaves them untouched (a checkpoint).  Synchronous.  DG_EINVAL, closing nothing,
 *        for a slot that is not open or listed twice, too small an output, or a stream in the "Cannot update unknown
 *        centers" state (as dg_multi_get_state reports it).
 *      dg_multi_import: opens n packed states (blob_host, blob_bytes in all) in the lowest free slots, in order, into
 *        slots_out.  Each continues its stream: the next dg_multi_step gives it the windows, results and names it would
 *        have had on its source.  The audio goes to the slot's ring and frames to its 16 kHz ring at absolute position
 *        mod their capacities, the history is written at this handle's history stride.  gals (null, or n entries, null
 *        meaning the handle's default gallery): the gallery of each state that was named from one, named at the state's
 *        own threshold; it must outlive the slot.  One copy, one launch per round.  Synchronous.  DG_EINVAL, naming the
 *        state and the reason, opening nothing and launching nothing, for: another format version or kind, other windows,
 *        F, K, D, M, gamma, beta or normalize_weights, a source rate this handle did not declare, more buffers than the
 *        handle's num_windows, audio beyond the ring's capacity, a clustering state that failed on its source, a state named
 *        from a gallery without one (or one of another size, dimension or device), a malformed state, or too few free
 *        slots.  Both calls keep a device staging buffer and a pinned buffer of up to 256 MiB of states (plus the piece
 *        list) for the handle's life once a move needed them; the call that first grows them synchronises the device.
 *        The gaps that align the sections are zero, so a state's bytes depend on the stream alone. ---- */
int dg_multi_export_bytes(const dg_multi* h, const int32_t* slots, int n, int64_t* bytes_out);
int dg_multi_export(dg_multi* h, const int32_t* slots, int n, int close, void* out_host, int64_t out_bytes);
int dg_multi_import(dg_multi* h, const void* blob_host, int64_t blob_bytes, int n, dg_gallery* const* gals,
                    int32_t* slots_out);
/* test hook (host only, no GPU): dg_multi_export of one stream of a VAD handle and dg_multi_import of its state into another
 * with other slots, max_windows_per_stream and num_windows, the pieces run on the host; see csrc/api_multi.cu. */
int dg_selftest_multi_transfer_host(const int32_t* geom, int n_ops, const int32_t* ops, const float* samples_host,
                                    int32_t* result, int src_slot, int patch, float* ring_out, float* yring_out, float* hist_out,
                                    int64_t cap, int64_t* info, char* message, int msg_cap);
/* test hook (host only, no GPU): dg_multi's tick planning for `slots` streams with pipeline windows of out_chunk / out_step
 * samples and the declared rates rates int32 [n_rates][5] = {o, n, w, chunk, step} (refused as dg_multi_add_rate refuses
 * them, DG_EINVAL).  ops int32 [n_ops][3] = {kind, slot, n}: 0 open slot at rate id n (-1: the pipeline's rate), 1 close slot,
 * 2 push n samples, 4 tick.  result int32 [n_ops]: each op's return code.  records int64 [cap][5] = {tick, kind, slot, a, b},
 * *n_records of them: kind 0 a resampling item (16 kHz frames [a, a + b) of the stream), kind 1 a window of the tick (it
 * starts at source sample a, batch row b).  DG_EINVAL if more than cap records. */
int dg_selftest_multi_frames_host(int slots, int max_wps, int out_chunk, int out_step, int n_rates, const int32_t* rates,
                                  int n_ops, const int32_t* ops, int32_t* result, int64_t* records, int cap, int* n_records);
/* test hook (host only, no GPU): dg_multi's bookkeeping of pushed audio on `slots` rings of C samples, with ring_scatter's
 * writes done on the host.  ops int32 [n_ops][3] = {kind, slot, n}: 0 open slot, 1 close slot (its staged samples are
 * dropped), 2 push the next n samples of samples_host (a refused push still skips them), 3 consume n samples (as a tick's
 * windows do), 4 tick (every staged sample to its ring).  result int32 [n_ops]: each op's return code, DG_EINVAL for a
 * refused one (a push beyond the ring capacity, a closed or unknown slot).  rings_host float [slots][C]: written by ticks. */
int dg_selftest_multi_staging_host(int slots, int C, int n_ops, const int32_t* ops, const float* samples_host, int32_t* result,
                                   float* rings_host);
/* test hook (host only, no GPU): the plan of a tick's grouped gallery search.  slots int32 [n][3] = {slot, gallery key (-1:
 * none), unnamed speakers} of the tick's slots in slot order; G int32 [n_keys] and thr [n_keys] the galleries' sizes and
 * thresholds.  Outputs: groups int32 [n][6] = {key, G, tiles, per_split, splits, query upper bound} in order of each key's
 * first slot, segs int32 [n][2] = {slot, group} group by group, work int32 [cap][3] = {group, query tile, split} (the CTAs of
 * gallery_nearest, split-major), counts int32 [4] = {groups, segments, work items, largest split count}.  DG_EINVAL if
 * more than cap work items. */
int dg_selftest_gallery_plan_host(int n, const int32_t* slots, int n_keys, const int32_t* G, const double* thr,
                                  int32_t* groups_out, int32_t* segs_out, int32_t* work_out, int cap, int32_t* counts);
/* test hook (host only, no GPU): dg_multi_set_slot_gallery and dg_multi_set_names on a diarization handle of `slots` slots,
 * embeddings of dimension D and M speakers on device 0 that owns no device memory.  gal int32 [n_gal][3] = {G, D, device}
 * describe galleries (no entries).  ops double [n_ops][4] = {kind, slot, arg, x}: 0 open the slot (no default gallery),
 * 1 dg_multi_set_slot_gallery(slot, gallery arg or null for -1, threshold x), 2 give the slot gallery arg (host state only),
 * 3 dg_multi_set_names(slot, named = arg, speaker 0 claiming entry x), 4 the slot has had a tick, 5 close the slot.
 * result int32 [n_ops]: each op's return code; messages: each op's error message ("" when none), one per line.  Meant
 * for refusals: an accepted call 1 or 3 goes on to the device. */
int dg_selftest_multi_gallery_host(int slots, int D, int M, int n_gal, const int32_t* gal, int n_ops, const double* ops,
                                   int32_t* result, char* messages, int msg_cap);
/* ---- many live streams of the reference's VoiceActivityDetection (src/diart/blocks/vad.py:139-191: the segmentation
 *      network, the max over the local speakers, DelayedAggregation(hamming) and Binarize(tau_active), turns labelled
 *      "speech"), served as dg_multi serves SpeakerDiarization.
 *      dg_multi_create_vad: a dg_multi without an embedding model or clustering state.  Arguments as dg_multi_create's;
 *        tau = tau_active.  DG_EINVAL, naming dg_multi_create_vad, allocating and launching nothing, unless chunk and step
 *        are positive multiples of 4 with step <= chunk, max_streams * max_windows_per_stream <= 65535, 1 <= num_windows
 *        <= 256, tau is finite, the model has at most 8 local speakers (classes) and the window at most 1023 frames.
 *      Every other dg_multi_* entry point works on it as on a diarization handle, with these differences.  dg_multi_open*
 *        resets the slot's rings and aggregation history only.  A tick runs the segmentation network alone (sub-batches of
 *        at most 256 windows on the model handle's two scratch lanes), then per chunk the speech curve -- the max over the K
 *        local speakers in float32 (torch.amax: a NaN propagates), aggregated over the stream's latency / step most recent
 *        chunks in float64 -- compared with > tau: the very arithmetic of dg_post_step with one speaker and the identity map
 *        on those max curves, so the turns are bit for bit those of a VoiceActivityDetection fed the stream one window per
 *        call.  header_host and turns_host as dg_multi_step (every turn's speaker is 0); seg_dev receives the tick's scores
 *        [n_rows, F, K]; emb_dev and map_dev must be null, else DG_EINVAL.
 *      Memory per slot: its ring(s) as dg_multi_create, and a history of 2 (num_windows - 1) F floats. ---- */
int dg_multi_create_vad(dg_seg* seg, int chunk_samples, int step_samples, int max_streams, int max_windows_per_stream,
                        double tau, int num_windows, const double* hamming_host, dg_multi** out);

/* ---- resampling: torchaudio's T.Resample(orig, new) with its defaults (sinc_interp_hann, lowpass_filter_width 6,
 *      rolloff 0.99), what the reference's blocks.Resample applies to every window of a source at another rate (reference
 *      src/diart/blocks/utils.py:62-89, inference.py:101-123).  With g = gcd(orig, new), o = orig / g, n = new / g:
 *        y[r n + p] = sum_k x[r o + k - width] taps[p][k],  x = 0 outside the window,  output length ceil(n L / o).
 *      taps_host float32 [n][2 width + o] = torchaudio.functional.functional._get_sinc_resample_kernel (bit-identical;
 *      diart_b200.operators.sinc_resample_kernel builds it); width must be torchaudio's for the two rates. ---- */
typedef struct dg_resample dg_resample;
int dg_resample_create(int orig_rate, int new_rate, const float* taps_host, int width, int device, dg_resample** out);
/* output samples of an L-sample window, -1 on bad arguments */
int64_t dg_resample_out_len(const dg_resample* h, int64_t num_samples);
/* per-window form: in_dev [B, L] -> out_dev [B, dg_resample_out_len(h, L)], stream-ordered */
int dg_resample_forward(dg_resample* h, const float* in_dev, int B, int64_t L, float* out_dev, void* stream);
int dg_resample_destroy(dg_resample* h);
/* dg_stream_create for a source at the resampler's original rate (no multiple-of-4 rule): chunk, step, push_host and
 * available count source-rate samples (rearrange_audio_stream at the source rate); dg_stream_windows returns the windows
 * resampled, [B, dg_resample_out_len(rs, chunk)].  When step % o == 0 every output of the batch's unique source samples is
 * computed once and only the frames whose taps cross a window edge are recomputed per window; otherwise each window is
 * resampled from the ring.  Both give the same bits as dg_resample_forward on the stacked source windows.  The stream
 * borrows `rs`.  dg_pipeline_submit_stream / call_stream take such a stream like any other, with the per-window form of the
 * sinc layer (resampled windows are not exact hops of one stream at their edges). */
int dg_stream_create_resampled(int chunk_samples, int step_samples, dg_resample* rs, int max_windows, int device,
                               dg_stream** out);
/* resampled stream only: outputs [first, first + count) of window `window` (0 = first window since create / reset) for n
 * ranges_host int64 [n][3] = {window, first, count}, packed into out_host; bit-identical to those of dg_stream_windows.  The
 * window's source samples must still be in the ring (it was formed by the last dg_stream_windows / pipeline call, and nothing
 * was pushed since).  Synchronous. */
int dg_stream_crop_host(dg_stream* h, int n, const int64_t* ranges_host, float* out_host);

/* number of kernels launched by this library since load (bench.py's gpu_launches) */
int64_t dg_launch_count(void);
/* per-kernel CUDA-event timing on the launching stream (bench.py's roofline leg).  While enabled,
 * every kernel launch is bracketed by two events; dg_profile_report() synchronises the device and
 * writes {"kernel": {"count": n, "ms": total}, ...} into buf. */
int dg_profile_enable(int enable);
/* test hook: the same random shifted-window GEMM through the float32 reference kernel and the wgmma (fp16 hi/lo,
 * three products) kernel; epi 0 = bias -> f32, 1 = bias+leaky+bn -> fp16 hi/lo planes, 2 = bias+leaky+bn -> f32. */
int dg_selftest_gemm_tc(int M, int Cin, int KW, int dil, int N, int epi, float* max_abs_diff, float* out_rms);
/* test hook: one seeded wgmma GEMM with epilogue epi (0..5) under SM caps 0, 1, 3 and 7; *equal = 1 if every output (float32
 * rows, hi/lo planes, pooling partial sums) is byte-equal across the four grids.  epi 3: 3 x 3 Conv2d, KW = 9, dil = side
 * of the square zero-padded maps (M a multiple of dil^2); epi 4: 3 speakers, items of 296 rows; epi 5: N <= 64, items of
 * 888 rows (M a multiple of 888). */
int dg_selftest_gemm_tc_grid(int M, int Cin, int KW, int dil, int N, int epi, int* equal);
/* test hook: one seeded wgmma GEMM (one tap, epi 0..2) into outputs of pitch N + 40 with guard rows after M, all bytes preset
 * to a sentinel.  *outside_unchanged = 1 if no byte outside rows [0, M) x columns [0, N) changed, *equal = 1 if the rows
 * equal, byte for byte, those of the same GEMM written at pitch N, *refused = 1 if an output base off 16-byte alignment and
 * a pitch that is not a multiple of 16 bytes are both rejected with DG_EINVAL.  N a multiple of 4 (32 for epi 1). */
int dg_selftest_gemm_tc_bounds(int M, int Cin, int N, int epi, int* outside_unchanged, int* equal, int* refused);
/* test hook: one m64n8k16 wgmma per row shift r = 0..8 of its A descriptor into a 64B-swizzled TMA tile; bit r of
 * *ok_shifts is set if the product of rows r..r+63 is exact.  base_offset_mode 1 also sets the descriptor's matrix base
 * offset field to (start address >> 7) & 7, mode 0 leaves it 0. */
int dg_selftest_wgmma_row_shift(int base_offset_mode, unsigned* ok_shifts);
/* test hook: the same for the B operand, one m64n64k16 wgmma per row shift r = 0..8 of its B descriptor into a 64B-swizzled
 * TMA tile; bit r of *ok_shifts is set if the product with rows r..r+63 is exact. */
int dg_selftest_wgmma_b_row_shift(int base_offset_mode, unsigned* ok_shifts);
/* test hook: one seeded Conv1d GEMM (KW 2..9, Cin a multiple of 16 up to 128, epi 0, 1, 2 or 5) through the halo operand
 * mode (with and without an SM cap of 3) and the tap-box mode (Cin not a multiple of 64: taps folded into K through an
 * overlapping-row view, dil 1); *equal = 1 if all outputs are byte-equal, *halo = 1 if the shape takes the halo mode.
 * epi 5: N <= 64, items of 888 rows (M a multiple of 888). */
int dg_selftest_gemm_tc_halo(int M, int Cin, int KW, int dil, int N, int epi, int* equal, int* halo);
/* test hook: one seeded Conv1d with the MaxPool1d(3) epilogue (epi 5; KW 2..9, Cin a multiple of 16 up to 128, N <= 64,
 * items of 888 rows, M a multiple of 888) against the float32 reference GEMM pooled on the host: largest absolute
 * difference of the pooled rows and their rms; *ws = 1 if the launch took the weight-stationary kernel. */
int dg_selftest_gemm_tc_pool3_simt(int M, int Cin, int KW, int dil, int N, float* max_abs_diff, float* out_rms, int* ws);
/* test hook (host only, no GPU): the weight-side split of float32 values into the two IEEE fp16 operand planes
 * (hi = rn16(x), lo = rn16(x - hi), saturating).  What the device does to activations with cvt.rn.satfinite.f16.f32. */
int dg_selftest_split_f16_host(const float* x, long long n, unsigned short* hi, unsigned short* lo);
/* the ParamSincFB filter table the models are built with, from low_hz_ [40] and band_hz_ [40]: filters [251][80] (tap-major;
 * 40 cosine then 40 sine filters); host only */
int dg_selftest_sinc_filters_host(const float* low_hz, const float* band_hz, float* filters);
/* the kaldi fbank tables variant-B models are built with: frame_operator [514][400] (DC removal, pre-emphasis, Hamming window
 * and the 512-point real DFT; rows 0..256 real, 257..513 imaginary part) and mel_banks [80][257]; host only */
int dg_selftest_fbank_tables_host(float* frame_operator, float* mel_banks);
int dg_profile_report(char* buf, int cap);

/* ---- shared-identity mode (extension beyond the reference; SURVEY.md 8(e), BASELINE config 5): G ranks diarize
 *      independent streams against one table of global speakers.  Per pipeline step and rank:
 *        dg_cluster_export_delta -> record [M*D payload | M kinds | 2 reserved] float64 (what changed since the
 *        last merge); the host all-gathers the records (one NCCL all-gather, ~82 KB per rank);
 *        dg_cluster_merge applies all records in rank order with one deterministic rule (cluster.cu) so that all
 *        ranks hold bit-identical tables, and rewrites this rank's speaker maps of the step (maps_dev, n_maps
 *        int32 values) where a centre it created was merged into / moved to another index. ---- */
int dg_cluster_record_len(const dg_cluster* h);
int dg_cluster_export_delta(dg_cluster* h, double* record_dev, void* stream);
int dg_cluster_merge(dg_cluster* h, const double* records_dev /*[world, record_len]*/, int world, int rank,
                     int32_t* maps_dev /*nullable*/, int n_maps, void* stream);
/* The same exchange inside the pipelined flow (dg_pipeline_submit* / collect*): both calls are stream-ordered on the
 * pipeline's clustering stream, behind the clustering of every submitted step and ahead of the next one, so the protocol is
 * exactly the one-step-at-a-time protocol while the networks of the following steps keep running.
 *   dg_pipeline_identity_export: record_dev [record_len] float64 receives this rank's changes; `stream` waits for it
 *     (issue the all-gather on `stream`);
 *   dg_pipeline_identity_merge: the clustering stream waits for `stream`, merges, and relabels the maps of the steps
 *     clustered since the previous merge in their device slots (call the pair after every submit, before that step's collect). */
int dg_pipeline_identity_export(dg_pipeline* h, double* record_dev, void* stream);
int dg_pipeline_identity_merge(dg_pipeline* h, const double* records_dev, int world, int rank, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* DIART_B200_H */
