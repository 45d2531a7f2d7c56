// Resampling (dg_resample_*) and the device-side audio stream (dg_stream_*).
#include <string.h>

#include <algorithm>
#include <cmath>
#include <memory>
#include <numeric>

#include "host.cuh"

// ======================================================================== resampling
// torchaudio's T.Resample(orig, new) with its defaults (sinc_interp_hann, lowpass_filter_width 6, rolloff 0.99) -- what the
// reference's blocks.Resample applies to every window of a source at another rate (reference blocks/utils.py:62-89).  The taps
// come from the host (diart_b200.operators.sinc_resample_kernel), bit-identical to torchaudio's.
extern "C" int dg_resample_create(int orig, int new_rate, const float* kernel_host, int width, int device, dg_resample** out) {
  if (!out || !kernel_host || orig < 1 || new_rate < 1 || orig == new_rate) {
    set_error("dg_resample_create: rates must be positive and different, taps non-null");
    return DG_EINVAL;
  }
  const int gcd = std::gcd(orig, new_rate);
  RsGeom g;
  g.o = orig / gcd;
  g.n = new_rate / gcd;
  // torchaudio: width = ceil(lowpass_filter_width * orig / (min(orig, new) * rolloff)) on the reduced rates
  const double base = std::min(g.o, g.n) * 0.99;
  const int want = (int)std::ceil(6.0 * g.o / base);
  if (width != want) {
    set_error("dg_resample_create: taps of shape (" + std::to_string(g.n) + ", " + std::to_string(2 * width + g.o) +
              ") given, (" + std::to_string(g.n) + ", " + std::to_string(2 * want + g.o) + ") expected for " +
              std::to_string(orig) + " -> " + std::to_string(new_rate) + " Hz");
    return DG_EINVAL;
  }
  g.w = width;
  g.T = 2 * width + g.o;
  if (!resample_geom_ok(g)) {
    set_error("dg_resample_create: the reduced rate ratio " + std::to_string(g.o) + " / " + std::to_string(g.n) +
              " is too large for the resampling kernel");
    return DG_EINVAL;
  }
  DG_CUDA(cudaSetDevice(device));
  std::unique_ptr<dg_resample> h(new dg_resample());
  h->device = device;
  h->g = g;
  if (h->taps.ensure((size_t)g.n * g.T * 4)) return DG_ECUDA;
  DG_CUDA(cudaMemcpy(h->taps.p, kernel_host, (size_t)g.n * g.T * 4, cudaMemcpyHostToDevice));
  *out = h.release();
  return DG_OK;
}

extern "C" int64_t dg_resample_out_len(const dg_resample* h, int64_t num_samples) {
  if (!h || num_samples < 0) return -1;
  return resample_out_len(h->g, num_samples);
}

extern "C" int dg_resample_forward(dg_resample* h, const float* in_dev, int B, int64_t L, float* out_dev, void* stream) {
  if (!h || !in_dev || !out_dev || B < 1 || L < 1) {
    set_error("dg_resample_forward: bad arguments");
    return DG_EINVAL;
  }
  DG_CUDA(cudaSetDevice(h->device));
  const long long out_len = resample_out_len(h->g, L);
  RsJob j{};
  j.x = in_dev;
  j.base = RsItem{0, L, 0, out_len, 0};
  j.start_step = L;
  j.out_step = out_len;
  j.W = h->taps.as<float>();
  j.g = h->g;
  j.out = out_dev;
  return launch_resample(j, B, out_len, (cudaStream_t)stream);
}

extern "C" int dg_resample_destroy(dg_resample* h) {
  delete h;
  return DG_OK;
}

// the body of both constructors, after their own argument checks; rs: null, or the resampler of the windows
static int stream_create(int chunk_samples, int step_samples, dg_resample* rs, int max_windows, int device, dg_stream** out) {
  DG_CUDA(cudaSetDevice(device));
  std::unique_ptr<dg_stream> h(new dg_stream());
  h->device = device; h->S = chunk_samples; h->hop = step_samples; h->rs = rs;
  // room for the windows being read, a full batch being uploaded meanwhile, and the overlap tail
  h->C = ((chunk_samples + 2 * max_windows * step_samples + 1023) / 1024) * 1024;
  if (h->ring.ensure((size_t)h->C * 4) || h->pin.ensure((size_t)h->C * 4) || h->st.create() || h->e_up.create() ||
      h->e_read.create())
    return DG_ECUDA;
  DG_CUDA(cudaEventRecord(h->e_read, h->st));
  *out = h.release();
  return DG_OK;
}

extern "C" int dg_stream_create(int chunk_samples, int step_samples, int max_windows, int device, dg_stream** out) {
  if (!out || chunk_samples < 4 || step_samples < 4 || chunk_samples % 4 || step_samples % 4 || max_windows < 1 ||
      step_samples > chunk_samples) {
    set_error("dg_stream_create: chunk and step must be positive multiples of 4 samples, step <= chunk");
    return DG_EINVAL;
  }
  return stream_create(chunk_samples, step_samples, nullptr, max_windows, device, out);
}

// the same stream with its windows resampled by `rs` (borrowed): chunk and step count source-rate samples, in any number;
// dg_stream_windows returns [B, dg_resample_out_len(rs, chunk)] resampled windows
extern "C" int dg_stream_create_resampled(int chunk_samples, int step_samples, dg_resample* rs, int max_windows, int device,
                                          dg_stream** out) {
  if (!out || !rs || chunk_samples < 1 || step_samples < 1 || max_windows < 1 || step_samples > chunk_samples ||
      rs->device != device || resample_out_len(rs->g, chunk_samples) > (1 << 30)) {
    set_error("dg_stream_create_resampled: chunk and step must be positive, step <= chunk, resampler on the same device");
    return DG_EINVAL;
  }
  return stream_create(chunk_samples, step_samples, rs, max_windows, device, out);
}

// samples per window as dg_stream_windows returns them
int stream_window_len(const dg_stream* h) { return h->rs ? (int)resample_out_len(h->rs->g, h->S) : h->S; }

extern "C" int dg_stream_destroy(dg_stream* h) {
  delete h;
  return DG_OK;
}

extern "C" int dg_stream_reset(dg_stream* h) {
  if (!h) return DG_EINVAL;
  DG_CUDA(cudaSetDevice(h->device));
  DG_CUDA(cudaStreamSynchronize(h->st));
  h->wpos = h->rpos = 0;
  for (auto& e : h->inflight) h->spare.push_back(std::move(e.second));
  h->inflight.clear();
  return DG_OK;
}

// complete windows that have been pushed but not yet consumed
extern "C" int dg_stream_available(const dg_stream* h) {
  if (!h) return 0;
  const long long have = h->wpos - h->rpos;
  return have < h->S ? 0 : (int)((have - h->S) / h->hop + 1);
}

// appends n samples (host memory, any kind) to the stream; returns once they are staged (the upload is asynchronous)
extern "C" int dg_stream_push_host(dg_stream* h, const float* samples, int n) {
  if (!h || !samples || n < 0) {
    set_error("dg_stream_push_host: bad arguments");
    return DG_EINVAL;
  }
  if (h->wpos + n - h->rpos > h->C) {
    set_error("dg_stream_push_host: ring full (" + std::to_string(h->wpos - h->rpos) + " samples buffered, capacity " +
              std::to_string(h->C) + "): consume windows first");
    return DG_EINVAL;
  }
  DG_CUDA(cudaSetDevice(h->device));
  // samples older than rpos may be overwritten: uploads are ordered after the last kernel that read the ring
  DG_CUDA(cudaStreamWaitEvent(h->st, h->e_read, 0));
  // the mirror region [wpos, wpos + n) was last used by the uploads of samples one lap earlier: wait for those
  while (!h->inflight.empty() && h->inflight.front().first < h->wpos + n - h->C) {
    DG_CUDA(cudaEventSynchronize(h->inflight.front().second));
    h->spare.push_back(std::move(h->inflight.front().second));
    h->inflight.pop_front();
  }
  float* pin = h->pin.as<float>();
  int done = 0;
  while (done < n) {
    const int at = (int)((h->wpos + done) % h->C);
    const int len = std::min(n - done, h->C - at);
    memcpy(pin + at, samples + done, (size_t)len * 4);
    DG_CUDA(cudaMemcpyAsync(h->ring.as<float>() + at, pin + at, (size_t)len * 4, cudaMemcpyHostToDevice, h->st));
    done += len;
  }
  Event ev;
  if (!h->spare.empty()) {
    ev = std::move(h->spare.back());
    h->spare.pop_back();
  } else if (ev.create()) {
    return DG_ECUDA;
  }
  DG_CUDA(cudaEventRecord(ev, h->st));
  h->inflight.emplace_back(h->wpos, std::move(ev));
  h->wpos += n;
  DG_CUDA(cudaEventRecord(h->e_up, h->st));
  return DG_OK;
}

// materialises the next B windows as a dense [B, S] batch on `st` and advances the stream by B steps
int stream_expand(dg_stream* h, int B, float* wav_dev, cudaStream_t st) {
  if (dg_stream_available(h) < B) {
    set_error("dg_stream: " + std::to_string(B) + " windows requested, " + std::to_string(dg_stream_available(h)) + " available");
    return DG_EINVAL;
  }
  DG_CUDA(cudaStreamWaitEvent(st, h->e_up, 0));
  int rc;
  if (h->rs) {
    const RsGeom& g = h->rs->g;
    const long long out_len = resample_out_len(g, h->S);
    // ys is rewritten: the previous batch, possibly formed on another stream, must have been read
    DG_CUDA(cudaStreamWaitEvent(st, h->e_read, 0));
    if (h->hop % g.o == 0) {   // stream form: window b's inner outputs are the stream's outputs
      const long long nr = (long long)(B - 1) * (h->hop / g.o) + (out_len + g.n - 1) / g.n;
      if (h->ys.ensure((size_t)nr * g.n * 4)) return DG_ECUDA;
      if ((rc = launch_resample_stream(h->ring.as<float>(), h->C, h->rpos, h->hop, h->S, B, h->rs->taps.as<float>(), g,
                                       h->ys.as<float>(), wav_dev, st)))
        return rc;
    } else {                   // per-window form, straight from the ring
      RsJob j{};
      j.x = h->ring.as<float>();
      j.C = h->C;
      j.base = RsItem{h->rpos, h->S, 0, out_len, 0};
      j.start_step = h->hop;
      j.out_step = out_len;
      j.W = h->rs->taps.as<float>();
      j.g = g;
      j.out = wav_dev;
      if ((rc = launch_resample(j, B, out_len, st))) return rc;
    }
  } else {
    if (h->rpos % 4) {
      set_error("dg_stream: window start is not 16-byte aligned");
      return DG_EINVAL;
    }
    if ((rc = launch_expand_windows(h->ring.as<float>(), h->rpos, h->C, h->hop, h->S, B, wav_dev, st))) return rc;
  }
  DG_CUDA(cudaEventRecord(h->e_read, st));
  h->rpos += (long long)B * h->hop;
  return 0;
}

extern "C" int dg_stream_windows(dg_stream* h, int B, float* wav_dev, void* stream) {
  if (!h || !wav_dev || B < 1) {
    set_error("dg_stream_windows: bad arguments");
    return DG_EINVAL;
  }
  DG_CUDA(cudaSetDevice(h->device));
  return stream_expand(h, B, wav_dev, (cudaStream_t)stream);
}

// outputs [first, first + count) of resampled window `window` (counted from the stream's start or last reset), for n
// ranges {window, first, count}, packed into out_host; the window's source samples must still be in the ring.  Every output
// is computed as in dg_stream_windows, so the values are bit-identical to the windows'.  Synchronous.
extern "C" int dg_stream_crop_host(dg_stream* h, int n, const int64_t* ranges_host, float* out_host) {
  if (!h || !h->rs || n < 0 || (n && (!ranges_host || !out_host))) {
    set_error("dg_stream_crop_host: bad arguments (a resampled stream is required)");
    return DG_EINVAL;
  }
  if (!n) return DG_OK;
  const long long out_len = resample_out_len(h->rs->g, h->S);
  std::vector<RsItem> items((size_t)n);
  long long total = 0, max_cnt = 1;
  for (int i = 0; i < n; ++i) {
    const long long win = ranges_host[3 * i], lo = ranges_host[3 * i + 1], cnt = ranges_host[3 * i + 2];
    const long long start = win * h->hop;
    if (win < 0 || lo < 0 || cnt < 0 || lo + cnt > out_len) {
      set_error("dg_stream_crop_host: range " + std::to_string(i) + " lies outside the window");
      return DG_EINVAL;
    }
    if (start < h->wpos - h->C || start + h->S > h->wpos) {
      set_error("dg_stream_crop_host: window " + std::to_string(win) + " is not (or no longer) in the ring");
      return DG_EINVAL;
    }
    items[i] = RsItem{start, h->S, lo, cnt, total};
    total += cnt;
    max_cnt = std::max(max_cnt, cnt);
  }
  DG_CUDA(cudaSetDevice(h->device));
  if (h->crop_items.ensure(items.size() * sizeof(RsItem)) || h->crop_out.ensure((size_t)std::max(total, 1LL) * 4) ||
      h->crop_pin.ensure(std::max(items.size() * sizeof(RsItem), (size_t)total * 4)))
    return DG_ECUDA;
  memcpy(h->crop_pin.h, items.data(), items.size() * sizeof(RsItem));
  DG_CUDA(cudaMemcpyAsync(h->crop_items.p, h->crop_pin.h, items.size() * sizeof(RsItem), cudaMemcpyHostToDevice, h->st));
  RsJob j{};
  j.x = h->ring.as<float>();
  j.C = h->C;
  j.items = h->crop_items.as<RsItem>();
  j.W = h->rs->taps.as<float>();
  j.g = h->rs->g;
  j.out = h->crop_out.as<float>();
  int rc;
  if ((rc = launch_resample(j, n, max_cnt, h->st))) return rc;
  DG_CUDA(cudaMemcpyAsync(h->crop_pin.h, h->crop_out.p, (size_t)total * 4, cudaMemcpyDeviceToHost, h->st));
  DG_CUDA(cudaStreamSynchronize(h->st));
  memcpy(out_host, h->crop_pin.h, (size_t)total * 4);
  return DG_OK;
}
