// Shared declarations for the diart_b200 CUDA translation units (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include <atomic>
#include <string>
#include <vector>

namespace dg {

// ------------------------------------------------------------------ error plumbing
void set_error(const std::string& msg);
extern std::atomic<long long> g_launches;
// persistent kernels size their grid to the SM count; while two streams overlap (fused pipeline) the
// kernels of the lower-priority stream are capped so that they never wait for SMs held by the other one
extern thread_local int g_sm_limit;
inline int usable_sms() {
  int dev = 0, sms = 132;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  return (g_sm_limit > 0 && g_sm_limit < sms) ? g_sm_limit : sms;
}

#define DG_CUDA(expr)                                                                   \
  do {                                                                                  \
    cudaError_t _e = (expr);                                                            \
    if (_e != cudaSuccess) {                                                            \
      dg::set_error(std::string(#expr) + ": " + cudaGetErrorString(_e));                \
      return -2;                                                                        \
    }                                                                                   \
  } while (0)

// cudaFuncSetAttribute is per DEVICE: `flags` is a function-local static bool[64]; returns true the first time it is asked
// about the current device (the caller then sets the attribute)
inline bool first_use_on_device(bool* flags) {
  int dev = 0;
  cudaGetDevice(&dev);
  if (dev < 0 || dev >= 64) return true;
  if (flags[dev]) return false;
  flags[dev] = true;
  return true;
}

// every kernel launch goes through this so bench.py can report `gpu_launches`
#define DG_LAUNCHED()                                                                   \
  do {                                                                                  \
    dg::g_launches.fetch_add(1, std::memory_order_relaxed);                             \
    cudaError_t _e = cudaGetLastError();                                                \
    if (_e != cudaSuccess) {                                                            \
      dg::set_error(std::string("kernel launch failed at ") + __FILE__ + ":" +          \
                    std::to_string(__LINE__) + ": " + cudaGetErrorString(_e));          \
      return -2;                                                                        \
    }                                                                                   \
  } while (0)

// per-kernel CUDA-event timing (bench.py's roofline leg): when enabled through dg_profile_enable(),
// every launcher brackets its launch with two events on the launching stream.
struct ProfScope {
  bool on;
  cudaStream_t st;
  cudaEvent_t a, b;
  const char* name;
  long long first = 0;
  ProfScope(const char* name, cudaStream_t st);
  ~ProfScope();
};

// ------------------------------------------------------------------ geometry of the path
// 80000 samples -> sinc(k251,s10) 7975 -> pool3 2658 -> k5 2654 -> pool3 884 -> k5 880 -> pool3 293.
// Activations are stored time-major / channels-last, [item][row][channel], with a fixed row
// stride per item that is divisible by 9 so that the two pool-by-3 stages keep rows aligned:
// a conv layer is then a pure shifted-window GEMM over the flattened [B*stride, C] matrix and
// rows past an item's valid length are harmless finite garbage that no consumer reads.
struct Geom {
  int S;        // samples per chunk
  int T0c;      // sinc conv outputs              (7975)
  int T0;       // after pool                      (2658)
  int T1;       // conv1+pool valid                (884)
  int T2;       // conv2+pool valid = frames       (293)
  int S0, S1, S2;  // row strides per item         (2664, 888, 296)
};
inline Geom make_geom(int S) {
  Geom g;
  g.S = S;
  g.T0c = (S - 251) / 10 + 1;
  g.T0 = g.T0c / 3;
  g.T1 = (g.T0 - 4) / 3;
  g.T2 = (g.T1 - 4) / 3;
  g.S2 = g.T2 + 3;                      // >= T2, room for pool alignment
  while ((g.S2 * 9) < g.T0 + 0 || (g.S2 * 3) < g.T1) g.S2++;
  g.S1 = g.S2 * 3;
  g.S0 = g.S1 * 3;
  return g;
}

__device__ __forceinline__ float leaky(float x) { return x > 0.f ? x : 0.01f * x; }

// ------------------------------------------------------------------ launchers (defined per .cu)
// sincnet.cu
int launch_wave_stats(const float* wav, int B, int S, float* mean, float* rstd, cudaStream_t st, const int* skip_flag = nullptr);
bool stream_stats_ok(int S, int hop);
size_t stream_stats_doubles(int B, int S, int hop);
int launch_stream_stats(const float* wav, int B, int S, int hop, double* part, float* mean, float* rstd, const int* flag,
                        cudaStream_t st);
int launch_instnorm_stats(const float* x, int B, int stride_rows, int T, int C, int ldc, const float* gamma,
                          const float* beta, float* sc, float* sh, cudaStream_t st, int pool = 0, const int* skip_flag = nullptr);
int launch_instnorm_finalize(const float* part, int B, int item_rows, int tile_rows, int T, int C, int N, const float* bias,
                             const float* gamma, const float* beta, float* sc, float* sh, int ld, cudaStream_t st);
// gemm.cu -- float32 reference GEMM of the wgmma self-test (dg_selftest_gemm_tc)
enum Epi { EPI_BIAS = 0, EPI_BIAS_LEAKY_BN = 2 };
struct GemmArgs {
  const float* A;      // [Mrows_in, lda]
  int lda;             // channel stride of A (>= Cin)
  int Cin;             // channels consumed per tap (multiple of 4)
  int KW, dil;         // taps, dilation (rows)
  long long Mtot;      // rows of A that exist (reads past it return 0)
  long long M;         // output rows to produce
  const float* W;      // [KW*Cin, ldw]
  int ldw;             // column stride of W (>= N, multiple of 4)
  int N;               // valid output channels
  const float* bias;   // [N] or null
  const float* bn_scale;  // [N] (EPI_BIAS_LEAKY_BN)
  const float* bn_shift;
  float* C;            // [M, ldc]
  int ldc;
  int epi;
  const char* tag;   // kernel label for profiling (layer name)
};
int launch_gemm(const GemmArgs& a, cudaStream_t st);
// gemm_tc.cu -- wgmma / TMA path (hi/lo split precision, three products)
constexpr int TC_POOL_SLOTS = 9, TC_POOL3_SLOTS = 3;   // pool_part values per (tile, item, column) of epi 4 / epi 5
struct TcGemm {
  const void* A_hi;    // fp16 [Mtot, lda]
  const void* A_lo;
  int lda, Cin, KW, dil;
  long long Mtot, M;
  const void* W_hi;    // fp16 [Npad, KW*Cin]  (n-major: row n holds its K weights, tap-major)
  const void* W_lo;
  float w_scale;       // power-of-two factor the W planes were multiplied by (0 = 1): undone on the accumulator
  int Npad, N;
  const float* bias;
  const float* bn_scale;
  const float* bn_shift;
  float* out_f32;      // [M, ldc] (float32 epilogues)
  void* out_hi;        // fp16 [M, ldc] (split epilogue)
  void* out_lo;
  int ldc;
  int epi;             // 0 bias -> f32, 1 bias+leaky+bn -> hi/lo planes, 2 bias+leaky+bn -> f32, 3 conv2d (see below)
  const char* tag;
  const int* tap_off;  // host array [KW]: row offset of every tap; null = j * dil (Conv1d)
  // epi 3 (Conv2d on zero-padded channels-last maps, rows = (item, w, h) of a [Wp][Hp] map): BatchNorm2d affine (bn_scale,
  // bn_shift) -> + residual planes -> ReLU -> hi/lo planes (and / or float32) at the same position of the [Wop][Hop] map;
  // stride2: the convolution is evaluated at every centre and only the odd (w, h) are kept
  int Wp, Hp, Wop, Hop, stride2, relu;
  const void* res_hi;
  const void* res_lo;
  // epi 4 (TDNN5 + weighted statistics pooling, heads.cu: pool_finalize): bias -> LeakyReLU -> BatchNorm, then per 128-row tile
  // and item the sums  S1 = sum_t w_k[t] e,  S2 = sum_t w_k[t] e^2  of e = d - p, d = x - bn_shift, for the K local speakers,
  // around a pivot p: 0, or for a channel far from its BatchNorm shift the average of d at two of the item's valid rows
  const float* pool_w;   // [Mtot][4]
  float* pool_part;      // [m_tiles][2][TC_POOL_SLOTS][N]: [4][2] sums, then p
  int pool_item_rows, pool_K;
  int pool_T;            // valid rows of an item (the rows after them hold garbage and weight 0)
  // epi 5 (SincNet Conv1d + MaxPool1d(3) + InstanceNorm statistics): out_f32 = bias + max over row triplets ([M / 3, ldc]),
  // pool_part = per-tile partial sums [M / pool3_tile_rows][2][TC_POOL3_SLOTS][N] (sum and sum of squares of v - p, p = the
  // item's first pooled value in the tile, then p), reduced by launch_instnorm_finalize;
  // pool_item_rows = un-pooled rows per item (multiple of 3), pool3_T = valid pooled frames per item
  int pool3_T, pool3_tile_rows;
  int tap_boxes;         // 1: load A per tap even where the halo mode applies (self-tests compare the two operand paths)
};
// rows an m-tile of the pooling epilogue advances by: the largest multiple of 3 up to 126 that divides the item's rows
// (tiles never straddle items: an item's statistics are grouped identically wherever it sits in the batch); 0 if none >= 96
inline int gemm_tc_pool3_tile_rows(int item_rows) {
  for (int t = 126; t >= 96; t -= 3)
    if (item_rows % t == 0) return t;
  return 0;
}
int launch_gemm_tc(const TcGemm& g, cudaStream_t st);
bool gemm_tc_halo(const TcGemm& g);   // the launch loads each tile's rows once (halo mode) instead of once per tap
bool gemm_tc_ws(const TcGemm& g);     // epi 5: the weight-stationary kernel (W resident in shared memory, D^T = W . X^T)
// one wgmma per row shift r = 0..8 of its A descriptor (m64n8k16), or with `shift_b` of its B descriptor (m64n64k16), into a
// 64B-swizzled tile (dg_selftest_wgmma_row_shift, dg_selftest_wgmma_b_row_shift): bit r of *ok_shifts is set when the
// product with rows r..r+63 is exact for both k16 steps of the 32-channel row
int selftest_wgmma_row_shift(bool shift_b, int base_offset_mode, unsigned* ok_shifts);
int launch_split_ex(const float* x, long long rows_out, int C, int ld_in, int ld_out, int pool, int item_rows,
                    const float* sc, const float* sh, void* hi, void* lo, cudaStream_t st, const int* skip_flag = nullptr);
void split_weights_host(const float* w, int N, int Npad, int K, uint16_t* hi, uint16_t* lo, float scale = 1.f);
float weight_plane_scale(const float* w, size_t n);   // power of two that keeps the lo plane of small weights normal
uint16_t host_f32_to_h16(float f);
float host_h16_to_f32(uint16_t h);
// sinc_tc.cu -- SincNet stage 0 on wgmma (overlapping-row TMA view of the waveform)
int sinc_tc_rows_per_item(const Geom& g);
size_t sinc_tc_plane_elems(int B, const Geom& g);
void sinc_tc_pack_filters(const float* filt, uint16_t* planes /*[2][80][256]*/);
void sinc_tc_affine_consts(const float* filt, float beta, float* cf);
int launch_sinc_prep(const float* wav, const float* mean, const float* rstd, int B, const Geom& g, void* planes_hi,
                     void* planes_lo, cudaStream_t st, const int* skip_flag = nullptr);
int launch_sinc0_tc(float gamma, const float* cf_dev, const void* w_planes, int B, const Geom& g, const void* planes_hi,
                    const void* planes_lo, float* p0, cudaStream_t st, const int* skip_flag = nullptr);
// stream form of the sinc layer (sinc_tc.cu): the batch is B windows of one stream, `hop` samples apart
struct SincStreamGeom {
  int Ls;        // unique samples (B-1)*hop + S
  int P;         // conv positions of the stream
  int rows;      // rows of the overlapping-row view (one "item")
  size_t plane;  // elements per shifted copy
};
SincStreamGeom sinc_stream_geom(int B, const Geom& g, int hop);
int launch_overlap_check(const float* wav, int B, int S, int hop, int* flag, cudaStream_t st);
int launch_stream_prep(const float* wav, const float* rstd, int B, const Geom& g, int hop, void* planes_hi, void* planes_lo,
                       int* flag, cudaStream_t st);
int launch_sinc0_tc_stream(const void* w_planes, int B, const Geom& g, int hop, const void* planes_hi, const void* planes_lo,
                           float* craw, const int* flag, cudaStream_t st);
size_t sinc_pool_part_floats(int B, const Geom& g, int hop);
int launch_sinc_pool_fused(const float* craw, const float* mean, const float* rstd, const float* cf, const float* hsum, float gamma,
                           int B, const Geom& g, int hop, const float* g0, const float* b0, float* part, float* sc, float* sh,
                           void* planes_hi, void* planes_lo, const int* flag, cudaStream_t st);
// lstm_tc.cu -- recurrence on wgmma (W_hh hi plane in registers, lo plane in shared memory)
size_t lstm_tc_plane_elems();
int lstm_tc_rows(int B);   // batch rows per CTA of the recurrence at batch B (8 or 16)
int lstm_tc_ctas(int B);   // CTAs (= SMs) one recurrence launch occupies at batch B
float lstm_tc_pack_whh(const float* whh_fwd, const float* whh_bwd, uint16_t* hi, uint16_t* lo);   // -> plane scale
// hout (float32) and / or out_hi, out_lo (16-bit planes of the next GEMM's operand) receive h_t
int launch_lstm_layer_tc(const float* gx, const void* whh_hi, const void* whh_lo, float w_scale, int B, int T, int stride,
                         float* hout, void* out_hi, void* out_lo, cudaStream_t st);
// heads.cu
int launch_seg_final(const float* y /*[B*stride,128]*/, const float* wc /*[K][128]*/, const float* bc, int B, int T,
                     int stride, int K, float* seg /*[B,T,K]*/, cudaStream_t st);
int launch_seg_powerset(const float* y, const float* wc, const float* bc, int B, int T, int stride, int C, int num_speakers,
                        const unsigned* masks_dev, float* seg /*[B,T,num_speakers]*/, cudaStream_t st);
int launch_osp(const float* seg, int B, int F, int K, float gamma, float beta, int normalize, float* out,
               cudaStream_t st);
// OSP sets (sweeps over overlap-aware weightings): set g = {gamma[g], beta[g], normalize[g]}, passed by value
constexpr int DG_MAX_OSP_SETS = 64;
struct OspSets {
  float gamma[DG_MAX_OSP_SETS], beta[DG_MAX_OSP_SETS];
  int normalize[DG_MAX_OSP_SETS];
};
// one launch over (item, set): set g's weights [B,F,K] at out + g B F K, the bits launch_osp gives at that set
int launch_osp_sets(const float* seg, int B, int F, int K, const OspSets& sets, int G, float* out, cudaStream_t st);
int launch_stats_pool(const float* x /*[B*stride,C]*/, int B, int stride, int T, int C, const float* w /*[B,F,K]*/,
                      int F, int K, const int* idx0, const int* idx1, const float* lam1, float eps,
                      float* pooled /*[B*K, 2C]*/, cudaStream_t st, long long item_pitch = 0, int row_pitch = 0);
// fused pooling (epi 4 of gemm_tc): row weights + their sums, and the final mean / std from the per-tile partial sums
int launch_pool_weights(const float* w /*[B,F,K]*/, int B, int F, int K, int item_rows, int T, const int* idx0, const int* idx1,
                        const float* lam1, float eps, float* row_w /*[B*item_rows][4]*/, float* vsum /*[B*K][2]*/, cudaStream_t st);
// launch_pool_weights for G sets in one launch: set g reads w + g B F K, writes row_w + g rw_stride and vsum + g B K 2
int launch_pool_weights_sets(const float* w, int B, int G, int F, int K, int item_rows, int T, const int* idx0, const int* idx1,
                             const float* lam1, float eps, float* row_w, long long rw_stride, float* vsum, cudaStream_t st);
int launch_pool_finalize(const float* part, const float* row_w, const float* vsum, const float* pivot, int B, int K, int C,
                         int item_rows, int T, float eps, float* pooled /*[B*K][2C]*/, cudaStream_t st);
int launch_l2norm(const float* in, int rows, int D, float norm, float* out, cudaStream_t st);
int launch_row_equal_flags(const float* wav, int N, int S, int* flags, cudaStream_t st);
int launch_gather_rows(const float* src, const int* index, int rows, int cols, float* dst, cudaStream_t st);
// resnet.cu -- variant B of the embedding (WeSpeaker ResNet34): fbank front end and stem around the Conv2d GEMMs
// planes of s_b (x * 2^15 - p_b) per item b, with p_b and s_b from the item's range; inv_scale [B] receives 1 / s_b, level
// [B][S / 80] the value of every constant 80-sample piece (NaN for the others)
int launch_fb_planes(const float* wav, int B, int S, void* hi, void* lo, float* inv_scale, float* level, cudaStream_t st);
int launch_fb_mel(const float* spec, int ld, int rows_per_item, int T, int B, const float* inv_scale, const float* level,
                  const float* banks, const int* k_lo, const int* k_hi, float* logmel, cudaStream_t st);
int launch_fb_mean(const float* logmel, int B, int T, float* mean, cudaStream_t st);
int launch_rn_stem(const float* logmel, const float* mean, int B, int T, const float* w, const float* sc, const float* sh,
                   void* hi, void* lo, cudaStream_t st);
// cluster.cu
struct ClusterParams {
  int M, D;
  float tau_f, rho_f;   // thresholds as numpy compares them (float32, see cluster.cu)
  double delta;
  int metric;           // 0 cosine (default), 1 euclidean, 2 sqeuclidean, 3 cityblock, 4 chebyshev (scipy cdist names)
};
int launch_cluster_step(const ClusterParams& p, const float* seg, const float* emb, int B, int F, int K,
                        double* centers, int* active, int* initialized, float* prep /*scratch*/,
                        double* prep_d /*scratch*/, int32_t* map, float* permuted, cudaStream_t st);
int launch_cluster_export(const double* centers, const int* active, const double* base, const int* base_active, int M,
                          int D, double* record, cudaStream_t st);
int launch_cluster_merge(const double* records, int world, int rank, const ClusterParams& p, int rec_len, double* centers,
                         int* active, double* base, int* base_active, int* initialized, int32_t* relabel,
                         cudaStream_t st);
int launch_relabel_maps(int32_t* maps, int n, const int32_t* relabel, cudaStream_t st);
// states = (file, trial) pairs over the concatenated chunks of several files: file f owns chunks
// [chunk_off[f], chunk_off[f + 1]) of B; thresholds trials_dev [T][3] = {tau, rho, delta} float64; one CTA per entry of
// states_dev [S] {file, trial} (the launch order); state s = file * T + trial owns centers [s][M][D], active [s][32] and
// initialized [s][2]; maps [T][B][K].  own_rows (many streams, each at its own thresholds): trial only selects the row of
// trials_dev, state s = file owns the tables and every state writes maps [B][K]
int launch_cluster_sweep(const ClusterParams& p, const double* trials_dev, int T, const int2* states_dev, int S,
                         const int* chunk_off_dev, const float* seg, const float* emb, int B, int F, int K, double* centers,
                         int* active, int* initialized, float* prep, double* prep_d, int32_t* maps, cudaStream_t st,
                         bool own_rows = false);
// launch_cluster_sweep over the embeddings of G OSP sets, emb [G][B][K][D]: the prep pass runs over (chunk, set) into prep
// [G][B][K][3] / prep_d [G][B][K], and a state of trial t reads the embeddings and prep rows of set (int)trials_dev[t * 4 + 3]
// (trials_dev [T][4] = {tau, rho, delta, set})
int launch_cluster_sweep_sets(const ClusterParams& p, const double* trials_dev, int T, const int2* states_dev, int S,
                              const int* chunk_off_dev, const float* seg, const float* emb, int G, int B, int F, int K,
                              double* centers, int* active, int* initialized, float* prep, double* prep_d, int32_t* maps,
                              cudaStream_t st);
size_t cluster_prep_floats(int B, int K);
// the seeded start of nf * T sweep states (state s = f T + t, tables as launch_cluster_sweep, already zeroed): file f's known
// centroids are rows [seed_off[f], seed_off[f + 1]) of seeds [n][D]; state s gets them as centres 0 .. n_f - 1, active, and
// initialized [s][0] = 1 when n_f > 0 (dg_multi_open_seeded's state for a stream)
int launch_sweep_seed(const int* seed_off, const double* seeds, int nf, int T, int M, int D, double* centers, int* active,
                      int* initialized, cudaStream_t st);
// post.cu -- aggregation + binarisation + run-length turns (reference diarization.py:205-232) of the sweeps: Nv virtual chunks,
// virtual chunk c = real chunk vchunk[c] (vchunk null: chunk c) of the N whose scores seg [N][F][K] and maps [T][N][K] are
// given; header [T][Nv][4]; trial t thresholds at taus[t]
int launch_post_virtual(const float* seg, const int32_t* map, int N, const int32_t* vchunk, int Nv, int F, int K, int M, int nw,
                        const int32_t* plan, int plan_stride, const double* hamming, const double* taus, int T,
                        int32_t* header, uint32_t* turns, int turn_cap, unsigned int* total, cudaStream_t st);
int launch_expand_windows(const float* ring, long long r0, int C, int hop, int S, int B, float* wav, cudaStream_t st);
// post.cu -- live streams in one batch (dg_multi; dg_post is one stream).  A piece of the staging upload: n samples at
// staged[src] belong at absolute sample dst of slot `slot`.  A slot with windows in the batch: its n windows are rows [row0,
// row0 + n); its post-path history is copy `cur` of the two, with n_hist chunks, of which it keeps at most nw - 1 (nw = its
// stream's latency / step).
struct RingPiece {
  long long src, dst;
  int slot, n;
};
struct TickSlot {
  int slot, row0, n, cur, n_hist, nw, pad[2];
};
int launch_ring_scatter(const float* staged, const RingPiece* pieces, int n_pieces, int C, float* rings, cudaStream_t st);
// rows [B] = {entry of act, window index i within that slot's rows}; entry b = samples [start[b], start[b] + S) of its slot's
// ring, written to batch row act[rows[b].x].row0 + i (any subset of a tick's rows can be gathered)
int launch_ring_gather(const float* rings, int C, const TickSlot* act, const int2* rows, const long long* start, int S, int B,
                       float* wav, cudaStream_t st);
// nw: the largest latency / step of any slot (the history stride is nw - 1); params [n_act][3]: {tau, rho, delta} of each
// entry of act, float64 (the post-path reads tau)
int launch_post_slots(const float* seg, const int32_t* map, const float* hist_seg, const int32_t* hist_map,
                      const TickSlot* act, const int2* rows, int slots, int B, int F, int K, int M, int nw,
                      const int32_t* plan, int plan_stride, const double* hamming, const double* params, int32_t* header,
                      uint32_t* turns, int turn_cap, unsigned int* total, cudaStream_t st);
int launch_post_slots_history(const float* seg, const int32_t* map, float* hist_seg, int32_t* hist_map, const TickSlot* act,
                              int n_act, int slots, int F, int K, int nw, cudaStream_t st);
size_t cluster_prep_doubles(int B, int K);
// der.cu -- DER components of sweep trials over nf files (chunks [chunk_off[f], chunk_off[f + 1]) of N, timestamp shift
// shifts[f]).  Hypothesis segments: count per (file, trial, label) and scan into offsets [nf*T*M+1], then write
// [offsets[nf*T*M]][2] start / end (and, when segs_copy is given, the first copy_cap of them there too)
int launch_der_hyp_count(const int32_t* header, const uint32_t* turns, int nf, const int* chunk_off, int T, int N, int M,
                         const double* out_start, const double* out_res, const double* shifts, double collar, int* offsets,
                         cudaStream_t st);
int launch_der_hyp_write(const int32_t* header, const uint32_t* turns, int nf, const int* chunk_off, int T, int N, int M,
                         const double* out_start, const double* out_res, const double* shifts, double collar, int* offsets,
                         double* segs, double* segs_copy, int copy_cap, cudaStream_t st);
// reference of file f: R[f] labels, offsets roff [f][DER_ROFF] (R[f] + 1 used) into rseg [S][2];
// comp [nf][T][5] = {false alarm, missed, confusion, correct, total}.  With uoff (device [nf + 1]) the hypothesis of file f is
// cropped to its scored pieces useg [uoff[f], uoff[f + 1])[2] (sorted, apart by more than 1e-6 s, each truthy).  With named
// (device [nf][32]) the identification error: reference label r of file f is matched to hypothesis label named[f][r] (-1:
// none) instead of the optimal mapping
constexpr int DER_ROFF = 33;
int launch_der_score(const int* hoff, const double* hseg, int nf, int T, int M, const int* roff, const int* R,
                     const double* rseg, double* comp, cudaStream_t st, const int* uoff = nullptr,
                     const double* useg = nullptr, const int* named = nullptr);
// vad.cu -- VAD sweep: the speech curve of Nv chunks (max over K local speakers, aggregated as the post-path with one speaker;
// chunk c's frames at curve [curve_off[c], curve_off[c + 1])), chunk c = real chunk vchunk[c] of seg (vchunk null: chunk c);
// then per trial t the turns of curve > taus[t], header [T][N][4]
int launch_vad_curve_virtual(const float* seg, const int32_t* vchunk, int Nv, int F, int K, const int32_t* plan, int plan_stride,
                             const double* hamming, const long long* curve_off, double* curve, cudaStream_t st);
int launch_vad_binarize(const double* curve, const long long* curve_off, int N, int T, const double* taus, int32_t* header,
                        uint32_t* turns, int turn_cap, unsigned int* total, cudaStream_t st);
// vad.cu -- many live VAD streams (dg_multi): chunks grouped by slot as launch_post_slots, one speech curve per chunk, each
// slot's history of max curves hist_vad [2][slots][nw - 1][F]
int launch_vad_slots(const float* seg, const float* hist_vad, const TickSlot* act, const int2* rows, int slots, int B, int F,
                     int K, int nw, const int32_t* plan, int plan_stride, const double* hamming, const double* params,
                     int32_t* header, uint32_t* turns, int turn_cap, unsigned int* total, cudaStream_t st);
int launch_vad_slots_history(const float* seg, float* hist_vad, const TickSlot* act, int n_act, int slots, int F, int K, int nw,
                             cudaStream_t st);
// resample.cu -- polyphase sinc resampling (torchaudio's defaults): reduced ratio o / n, half-width w, T = 2w + o taps per phase
struct RsGeom {
  int o, n, w, T;
};
// one item = one window of source samples, x = 0 outside [start, start + len) (absolute sample indices, taken mod C for a
// ring); outputs [j_lo, j_lo + j_cnt) of it are written to out + out_off
struct RsItem {
  long long start, len, j_lo, j_cnt, out_off;
};
struct RsJob {
  const float* x;
  long long C;            // ring capacity, 0: x is a dense array
  const RsItem* items;    // device array, one per item, or null: item b = base shifted by b * start_step / b * out_step
  RsItem base;
  long long start_step, out_step;
  const float* W;         // [n][T]
  RsGeom g;
  float* out;
};
long long resample_out_len(const RsGeom& g, long long L);   // ceil(n L / o)
bool resample_geom_ok(const RsGeom& g);                     // the source span of one block fits in shared memory
// per-window form (and crops): `items` items, none with more than max_out outputs
int launch_resample(const RsJob& j, int items, long long max_out, cudaStream_t st);
// stream form (hop % o == 0): windows b = 0 .. B-1 of a ring start at rpos + b hop; ys: scratch of
// ((B-1) hop / o + ceil(out_len / n)) n floats; out [B][out_len]
int launch_resample_stream(const float* ring, long long C, long long rpos, long long hop, long long L, int B, const float* W,
                           const RsGeom& g, float* ys, float* out, cudaStream_t st);
// dg_multi's resampled streams.  A stream at a source rate keeps its source samples in a ring of stride C (sample t at t mod C)
// and its 16 kHz frames in a ring of Q frames (frame R at outputs [(R mod Q) n, (R mod Q) n + n), stride Y floats per slot).
// RsFrames: stream frames [first, first + count) of `slot`, all of whose taps are pushed samples; RsRow: the window of L source
// samples that starts at absolute sample `start` (= frame0 o) of `slot`, to batch row `row`.
struct RsFrames {
  long long first;
  int slot, count;
};
struct RsRow {
  long long start, frame0;
  int slot, row;
};
// the frames of every item (one launch; none with more than max_count frames)
int launch_resample_frames(const float* rings, long long C, const RsFrames* items, int n_items, long long max_count,
                           const float* W, const RsGeom& g, float* yrings, long long Y, long long Q, cudaStream_t st);
// the windows `rows` [n_rows] into wav [row][out_len]: interior frames r_lo .. r_hi from the 16 kHz rings, edge frames recomputed
int launch_resample_gather(const float* rings, long long C, const float* yrings, long long Y, long long Q, const RsRow* rows,
                           int n_rows, long long r_lo, long long r_hi, const float* W, const RsGeom& g, long long L,
                           long long out_len, float* wav, cudaStream_t st);

void fbank_frame_operator(std::vector<float>& op /*[514][400]*/);
void fbank_mel_banks(std::vector<float>& banks /*[80][257]*/, std::vector<int>& k_lo, std::vector<int>& k_hi);

// gallery.cu -- nearest-centroid search over speaker galleries, each E [Gp][Dp] float64 (rows >= G and columns >= D zero;
// Gp a multiple of GAL_TILE_E, Dp of GAL_KC, Dp the same for every gallery of a launch) with norms En [G].  A launch serves
// one or more groups, each one gallery at one threshold; a group's queries are one contiguous run.  A query q is row
// qd[q].x of X [*][D] (row stride D) in claim group qd[q].y; claim group r's claimed entries are claimed [r][32], indices
// into its group's gallery (-1: none; claimed null: no claims).  The cosine distance is 1 - clip(u.v / (|u| |v|), -1, 1) in
// float64.
constexpr int GAL_TILE_E = 64, GAL_TILE_Q = 128, GAL_KC = 16, GAL_NAME_PREFIX = 1024;
// A group of a launch: its gallery (E, En, G entries), threshold, and from gallery_plan its GAL_TILE_E-entry tiles split
// into `splits` runs of per_split tiles; q_ub an upper bound of its queries (host); its segments [seg0, seg1).
struct GalGroup {
  const double* E;
  const double* En;
  double threshold;
  int G, tiles, per_split, splits, q_ub, seg0, seg1, pad;
};
// one CTA of gallery_nearest: query tile `tile` of group `group` against split `split` of its gallery's tiles
struct GalWork {
  int group, tile, split;
};
int launch_gallery_norms(const double* E, int G, int Dp, double* En, cudaStream_t st);
// The grouped search plan: each group's tiles and splits, and the work list.  The split count is chosen over the query
// tiles of all groups (about two CTAs per SM in total, at most 64, at most a group's tiles); items are split-major, then
// group, then query tile, so one group is the grid (query tiles, splits).  Returns the largest split count (partials
// [splits][Qmax]).
int gallery_plan(std::vector<GalGroup>& groups, std::vector<GalWork>& work);
// per query and split of its group, the lexicographic minimum (distance, entry) over the unclaimed entries of the split:
// part_d / part_e [splits][Qmax] (+inf / -1 when none).  Group r's queries are [gq[r].x, gq[r].x + gq[r].y).
int launch_gallery_nearest(const GalGroup* groups, const GalWork* work, int n_work, const int2* gq, int Dp, const double* X,
                           int D, const int2* qd, int Qmax, const int32_t* claimed, double* part_d, int* part_e,
                           cudaStream_t st);
// the multi-stream queries of a tick: every active (active [slot][32]), unnamed (named [slot] bit g) global speaker g < M of
// the tick's segments segs [n] = {slot, group} (group by group, slots in order), in segment then g order, as
// qd = {slot M + g, slot}; seg_off [n + 1] its queries per segment, gq [group] = {offset, count} of each group's queries
// (groups [n_groups]: its segments); names [0] (the count of new names) reset to 0.
int launch_gallery_queries(const int2* segs, int n, const GalGroup* groups, int n_groups, const int* active,
                           const uint32_t* named, int M, int2* qd, int* seg_off, int2* gq, int* names, cudaStream_t st);
// One warp per segment [seg_off[s], seg_off[s + 1]) (at most 32 queries of one claim group) of group segs[s].y: each
// query's best over its group's splits; a candidate when distance < the group's threshold; among candidates for one entry the
// smallest (distance, position) wins.  entry_out / dist_out (standalone, may be null): per query the winner's entry or -1, and
// its best distance.  named non-null (streams): each winner g = qd.x mod M of claim group r sets named [r] bit g and claimed
// [r][g], and appends {r, g, entry} to list [.][3] at names [0]++ (the first GAL_NAME_PREFIX entries also to prefix [.][3]).
int launch_gallery_claim(const double* part_d, const int* part_e, int Qmax, const int2* qd, const int* seg_off,
                         const int2* segs, int n_seg, const GalGroup* groups, int32_t* claimed, int32_t* entry_out,
                         double* dist_out, uint32_t* named, int M, int* names, int32_t* list, int32_t* prefix, cudaStream_t st);

// transfer.cu -- n 32-bit words from src to dst: word i at src [(src_pos + i) mod src_mod] (src_mod 0: src [src_pos + i]),
// likewise for dst.  A ring piece is addressed by absolute position mod its ring's capacity on each side.
struct XferPiece {
  const uint32_t* src;
  uint32_t* dst;
  long long n, src_pos, src_mod, dst_pos, dst_mod;
};
// every piece in one launch (pieces is a device array); `tag` names the launch in the profile
int launch_slot_transfer(const XferPiece* pieces, int n_pieces, const char* tag, cudaStream_t st);

}  // namespace dg
