"""Device post-path of ``SpeakerDiarization.__call__`` (reference ``src/diart/blocks/diarization.py:205-232``):
``SpeakerMap.apply`` -> ``DelayedAggregation(step, latency, "hamming", "loose")`` -> ``Binarize(tau)`` run on the GPU
(``csrc/post.cu``); this module is the host half.

What stays on the host is what only the host knows -- time stamps.  ``SlidingWindow.crop(mode="loose", fixed=...)``
(pyannote.core; the shim in ``diart_b200/core.py`` has the same arithmetic) is float64 index arithmetic on chunk start
times: it is evaluated here, vectorised over the batch with exactly the reference's operation order, and handed to the
device as one small integer plan per chunk.  Everything that touches scores (permutation, Hamming-weighted average over
the ``latency / step`` most recent buffers, threshold, run-length encoding) happens on the device; one D2H brings back
the packed turn list, which is turned into ``Annotation`` objects here.
"""
from __future__ import annotations

import ctypes as C
from typing import List, Optional, Sequence, Tuple

import numpy as np
import torch

from .. import _lib
from ..core import Annotation, Segment, SlidingWindow, SlidingWindowFeature, extent_bounds


class DevicePostPath:
    def __init__(self, step: float, latency: float, tau: float, frames: int, local_speakers: int, max_speakers: int,
                 device: torch.device):
        assert step <= latency, "Invalid latency requested"
        self.step, self.latency, self.tau = float(step), float(latency), float(tau)
        self.F, self.K, self.M = int(frames), int(local_speakers), int(max_speakers)
        self.nw = int(round(latency / step))            # DelayedAggregation.num_overlapping_windows
        self.device = device
        self.labels = [f"speaker{g}" for g in range(self.M)]
        ham = np.ascontiguousarray(np.hamming(self.F), dtype=np.float64)
        h = C.c_void_p()
        _lib.check(_lib.lib().dg_post_create(self.F, self.K, self.M, self.nw, ham.ctypes.data, self.tau,
                                             device.index or 0, C.byref(h)))
        self._h = h
        self._hist_start = np.zeros(0)
        self._hist_res = np.zeros(0)
        self._turns = np.empty(1 << 16, dtype=np.uint32)

    def __del__(self):
        try:
            if getattr(self, "_h", None) is not None:
                _lib.lib().dg_post_destroy(self._h)
        except Exception:  # noqa: BLE001
            pass

    @property
    def handle(self) -> C.c_void_p:
        return self._h

    def reset(self):
        _lib.check(_lib.lib().dg_post_reset(self._h))
        self._hist_start = np.zeros(0)
        self._hist_res = np.zeros(0)

    # ------------------------------------------------------------------ the integer plan
    def plan(self, starts: np.ndarray, res: float):
        """starts (B,) float64 chunk start times, res = seconds per score frame of this batch ->
        (plan int32 (B, 4 + nw), out_start (B,), out_res (B,)); advances the buffer history by B chunks."""
        plan, out_start, out_res = post_plan(starts, res, self._hist_start, self._hist_res, self.nw, self.F, self.step,
                                             self.latency)
        B, H = len(starts), len(self._hist_start)
        s_all = np.concatenate([self._hist_start, starts])
        r_all = np.concatenate([self._hist_res, np.full(B, res)])
        keep = min(self.nw - 1, H + B)
        self._hist_start = s_all[len(s_all) - keep:] if keep else np.zeros(0)
        self._hist_res = r_all[len(r_all) - keep:] if keep else np.zeros(0)
        return plan, out_start, out_res

    # ------------------------------------------------------------------ results
    def buffers(self, B: int):
        need = turn_capacity(B, self.M, self.F)
        if len(self._turns) < need:
            self._turns = np.empty(need, dtype=np.uint32)
        return np.empty((B, 4), dtype=np.int32), self._turns

    def annotations(self, header: np.ndarray, turns: np.ndarray, n_turns: int, out_start: np.ndarray,
                    out_res: np.ndarray, shift: float = 0.0, uri: Optional[str] = None) -> List[Annotation]:
        """packed turns -> one Annotation per chunk, segments at frame middles (blocks/utils.py:45-58)"""
        return chunk_annotations(header, turns, n_turns, out_start, out_res, self.labels, shift, uri)

    def run(self, seg: torch.Tensor, maps: torch.Tensor, starts: np.ndarray, res: float, shift: float = 0.0):
        """device scores (B,F,K) + maps (B,K) -> list of Annotation (block-level entry; the fused pipeline uses
        dg_pipeline_call_host instead)"""
        return self.annotations(*self.turns(seg, maps, starts, res), shift)

    def turns(self, seg: torch.Tensor, maps: torch.Tensor, starts: np.ndarray, res: float):
        """``run`` up to the packed turns -> (header (B, 4), turns, n_turns, out_start (B,), out_res (B,))"""
        plan, out_start, out_res = self.plan(np.asarray(starts, dtype=np.float64), res)
        B = len(plan)
        header, turns = self.buffers(B)
        n = C.c_int()
        with torch.cuda.device(self.device):
            _lib.check(_lib.lib().dg_post_step(self._h, seg.data_ptr(), maps.data_ptr(), B, plan.ctypes.data,
                                               header.ctypes.data, turns.ctypes.data, len(turns), C.byref(n),
                                               _lib.stream_ptr(self.device)))
        return header, turns, n.value, out_start, out_res


def turn_capacity(B: int, speakers: int, frames: int) -> int:
    """the most turns B chunks can emit: up to frames + 1 output frames each (a stream's first chunk), every second one
    starting a turn of every speaker"""
    return B * speakers * ((frames + 2) // 2)


def post_plan(starts: np.ndarray, res: float, hist_start: np.ndarray, hist_res: np.ndarray, nw: int, F: int, step: float,
              latency: float):
    """The integer plan of dg_post_step for a batch of chunks starting at ``starts`` (B,) float64, ``res`` seconds per
    score frame, after the chunks of the history (``hist_start``, ``hist_res``: the last nw - 1 chunks seen, oldest first)
    -> (plan int32 (B, 4 + nw), out_start (B,), out_res (B,))."""
    B = len(starts)
    H = len(hist_start)
    s_all = np.concatenate([hist_start, starts])
    r_all = np.concatenate([hist_res, np.full(B, res)])
    c = np.arange(B)
    nb = np.minimum(H + c + 1, nw)
    # buffer j of chunk c (oldest first) is entry H + c - (nb - 1) + j of the concatenated history
    j = np.arange(nw)[None, :]
    idx = (H + c - (nb - 1))[:, None] + j
    valid = j < nb[:, None]
    idx = np.where(valid, idx, 0)
    return crop_plan(starts, np.full(B, res), s_all[idx], r_all[idx], nb, valid, nw, F, step, latency)


def crop_plan(starts: np.ndarray, res: np.ndarray, s_j: np.ndarray, r_j: np.ndarray, nb: np.ndarray, valid: np.ndarray,
              nw: int, F: int, step: float, latency: float):
    """The plan rows of chunks starting at ``starts`` (B,) with ``res`` (B,) seconds per score frame, whose aggregated
    buffers j (oldest first, ``valid`` (B, nw) for j < nb) start at ``s_j`` (B, nw) with resolution ``r_j`` (B, nw)
    -> (plan int32 (B, 4 + nw), out_start (B,), out_res (B,)).  The float64 arithmetic of the reference's
    ``SlidingWindow.crop(mode="loose", fixed=...)``, operation by operation."""
    end = starts + F * res                                  # buffers[-1].extent.end (duration == step)
    f_start = end - latency                                 # aggregation.py:216-217
    f_end = f_start + step
    fixed = np.where(f_end > f_start, f_end - f_start, 0.0)  # Segment.duration
    lo = np.ceil((f_start[:, None] - r_j - s_j) / r_j)      # SlidingWindow.crop, mode="loose"
    cnt = np.floor((fixed[:, None] + r_j) / r_j)            # SlidingWindow.samples(fixed, mode="loose")
    nf = cnt[:, 0]
    if np.any(valid & (cnt != nf[:, None])):
        raise ValueError("all input arrays must have the same shape")   # what np.stack raises in the reference
    plan = np.zeros((len(starts), 4 + nw), dtype=np.int32)
    plan[:, 0] = nb
    plan[:, 1] = nf
    plan[:, 4:] = np.where(valid, lo, 0)
    out_start, out_res = f_start.copy(), fixed / nf
    # first buffer of a stream: everything before the region is emitted too (aggregation.py:188-212)
    first = (nb == 1) & (starts == 0)
    if first.any():
        first_nf = np.floor((f_end + res) / res)            # crop of Segment(0, region.end), fixed = its duration
        plan[:, 2] = np.where(first, first_nf, 0)
        plan[:, 3] = np.where(first, np.ceil((0.0 - res - starts) / res), 0)
        out_start = np.where(first, 0.0, out_start)
        out_res = np.where(first, f_end / np.maximum(first_nf, 1), out_res)
    return plan, out_start, out_res


def turn_times(header: np.ndarray, turns: np.ndarray, n_turns: int, out_start: np.ndarray, out_res: np.ndarray,
               shift: float = 0.0):
    """packed turns -> (row of ``header`` each turn belongs to, speaker, on time, off time), segments at frame middles
    (blocks/utils.py:45-58).  ``header`` (R, 4) rows may be several states' headers over the same chunks (row r is chunk
    r % len(out_start))."""
    t = turns[:n_turns]
    # each row's turns are one contiguous block; sorted by offset the blocks tile [0, n_turns)
    order = np.argsort(header[:, 0], kind="stable")
    order = order[header[order, 1] > 0]
    row_of = np.repeat(order, header[order, 1])
    chunk_of = row_of % len(out_start)
    g = (t >> 20).astype(np.int64)
    on = ((t >> 10) & 1023).astype(np.float64)
    off = (t & 1023).astype(np.float64)
    s0, r0 = out_start[chunk_of], out_res[chunk_of]
    a = s0 + on * r0
    b = s0 + off * r0
    t_on = 0.5 * (a + (a + r0)) + shift                     # SlidingWindow[i].middle
    t_off = 0.5 * (b + (b + r0)) + shift
    return row_of, g, t_on, t_off


def chunk_turns(header: np.ndarray, turns: np.ndarray, n_turns: int, out_start: np.ndarray, out_res: np.ndarray, shift=0.0):
    """packed turns -> plain lists (offset and count per chunk, then speaker, on time, off time per turn), segments at frame
    middles (blocks/utils.py:45-58).  ``shift``: seconds added to every time stamp, one number or one per chunk."""
    per_chunk = np.ndim(shift) > 0
    row_of, g, t_on, t_off = turn_times(header, turns, n_turns, out_start, out_res, 0.0 if per_chunk else shift)
    if per_chunk:                                            # x + 0.0 + s == x + s: the same bits as a scalar shift
        s = np.asarray(shift, dtype=np.float64)[row_of]
        t_on, t_off = t_on + s, t_off + s
    return header[:, 0].tolist(), header[:, 1].tolist(), g.tolist(), t_on.tolist(), t_off.tolist()


def chunk_annotations(header: np.ndarray, turns: np.ndarray, n_turns: int, out_start: np.ndarray, out_res: np.ndarray,
                      labels: Sequence, shift=0.0, uri: Optional[str] = None) -> List[Annotation]:
    """packed turns -> one Annotation per chunk (row of ``header``), segments at frame middles (blocks/utils.py:45-58).
    ``labels``: the label of each global speaker, one list for every chunk or one list per chunk (streams with their own
    known speakers).  ``shift``: seconds added to every time stamp, one number or one per chunk (streams with their own
    shifts)."""
    B = len(header)
    offs, cnts, g, t_on, t_off = chunk_turns(header, turns, n_turns, out_start, out_res, shift)
    # the reference's shifted copy drops the modality
    modality = [("speech" if x == 0 else None) for x in np.asarray(shift).tolist()] if np.ndim(shift) > 0 else \
        [("speech" if shift == 0 else None)] * B
    per_chunk = B > 0 and not isinstance(labels[0], str)
    out = []
    for cidx in range(B):
        ann = Annotation(uri=uri, modality=modality[cidx])
        labels_c = labels[cidx] if per_chunk else labels
        o = offs[cidx]
        for i in range(o, o + cnts[cidx]):
            ann[Segment(t_on[i], t_off[i]), g[i]] = labels_c[g[i]]
        out.append(ann)
    return out


def aggregate_audio(chunk_buffer: List[SlidingWindowFeature], new: Sequence[SlidingWindowFeature], nw: int, step: float,
                    latency: float) -> Tuple[List[SlidingWindowFeature], List[SlidingWindowFeature]]:
    """``DelayedAggregation(step, latency, "first", "center")`` over the waveform buffers (reference
    diarization.py:76-77,228), for the whole batch: per chunk the crop of the OLDEST buffered waveform over the
    output region, as a view where the range lies inside the chunk.  The crop indices of all chunks are evaluated at once
    (numpy float64, the operation order of pyannote.core's ``crop(mode="center", fixed=...)``).
    Returns (outputs, new chunk_buffer)."""
    H, B = len(chunk_buffer), len(new)
    buf = list(chunk_buffer) + list(new)
    bounds = [extent_bounds(w) for w in new]
    w_start = np.array([b[0] for b in bounds])
    w_end = np.array([b[1] for b in bounds])
    first_idx = np.maximum(H + np.arange(B) + 1 - nw, 0) if nw > 1 else H + np.arange(B)     # oldest buffer of each chunk
    nbuf = np.minimum(H + np.arange(B) + 1, nw)
    sw0 = [buf[i].sliding_window for i in first_idx]
    s0 = np.array([sw.start for sw in sw0])
    d0 = np.array([sw.duration for sw in sw0])
    p0 = np.array([sw.step for sw in sw0])
    start = w_end - latency
    end = start + step
    fixed = np.where(end > start, end - start, 0.0)
    lo = np.rint((start - s0 - 0.5 * d0) / p0).astype(np.int64)          # SlidingWindow.closest_frame
    cnt = np.rint(fixed / p0).astype(np.int64)                           # SlidingWindow.samples(fixed, mode="center")
    is_first = ((nbuf == 1) & (w_start == 0)).tolist()
    # (plain Python numbers inside the per-chunk loop: indexing numpy arrays element by element costs more than the crops)
    first_l, lo_l, cnt_l, fixed_l, start_l = first_idx.tolist(), lo.tolist(), cnt.tolist(), fixed.tolist(), start.tolist()
    outs = []
    for c in range(B):
        first = buf[first_l[c]]
        data = first.data
        n = data.shape[0]
        if is_first[c]:
            # first buffer of a stream: [0, region.end) with the region pasted over its tail (aggregation.py:188-212)
            lo1 = int(np.rint((0.0 - s0[c] - 0.5 * d0[c]) / p0[c]))
            cnt1 = int(np.rint(end[c] / p0[c]))
            out = _crop(data, lo1, cnt1, n).copy()
            out[-cnt_l[c]:] = _crop(data, lo_l[c], cnt_l[c], n)
            res = end[c] / out.shape[0]
            outs.append(SlidingWindowFeature(out, SlidingWindow(start=0, duration=res, step=res)))
        else:
            out = _crop(data, lo_l[c], cnt_l[c], n)
            res = fixed_l[c] / out.shape[0]
            outs.append(SlidingWindowFeature(out, SlidingWindow(start=start_l[c], duration=res, step=res)))
    keep = min(nw - 1, H + B)
    return outs, (buf[len(buf) - keep:] if keep else [])


def resampled_stream_audio(stream, first: int, B: int, nw: int, step: float, latency: float) -> List[SlidingWindowFeature]:
    """``aggregate_audio`` for chunks ``first .. first + B - 1`` of a resampled ``DeviceAudioStream`` whose windows were just
    formed on the device and never copied back.  Chunk c crops its oldest buffered window, window max(c + 1 - nw, 0) of the
    stream, with the arithmetic of ``aggregate_audio``; the windows of this batch are all some chunk's oldest until
    ``nw - 1`` chunks later, so their crops for later chunks are fetched now and kept on the stream.  Only the cropped
    ranges (about one step of audio per chunk) come back from the device."""
    n, res = stream.window_samples, stream.window_resolution
    stash = stream.audio_stash
    todo = {}                                          # chunk -> (oldest window, lo, cnt, lo1, cnt1 or None, start, end, fixed)
    for c in range(first, first + B + nw - 1):
        o = max(c + 1 - nw, 0) if nw > 1 else c
        if c in stash or not (first <= o < first + B):
            if c < first + B and c not in stash:
                raise ValueError(f"chunk {c} needs window {o}, which is no longer on the device")
            continue
        s0 = stream.window_start_time(o)                # d0 = p0 = res: the window's SlidingWindow
        w_start = stream.window_start_time(c)
        w_end = w_start + n * res
        start = w_end - latency
        end = start + step
        fixed = end - start if end > start else 0.0
        lo = int(np.rint((start - s0 - 0.5 * res) / res))
        cnt = int(np.rint(fixed / res))
        nbuf = min(c + 1, nw)
        lo1 = cnt1 = None
        if nbuf == 1 and w_start == 0:
            lo1 = int(np.rint((0.0 - s0 - 0.5 * res) / res))
            cnt1 = int(np.rint(end / res))
        todo[c] = (o, lo, cnt, lo1, cnt1, start, end, fixed)
    ranges = []
    for c, (o, lo, cnt, lo1, cnt1, *_) in todo.items():
        spans = [(lo, cnt)] + ([(lo1, cnt1)] if lo1 is not None else [])
        a = min(min(max(l, 0), n - 1) for l, _ in spans)
        b = max(min(max(l + k - 1, 0), n - 1) for l, k in spans) + 1
        ranges.append((o, a, b - a))
    flat = stream.crops(ranges) if ranges else np.zeros(0, np.float32)
    off = 0
    for (c, (o, lo, cnt, lo1, cnt1, start, end, fixed)), (_, a, k) in zip(todo.items(), ranges):
        piece = flat[off:off + k, None]
        off += k

        def crop(l, m):
            if l >= 0 and l + m <= n:
                return piece[l - a:l - a + m]
            return piece[np.clip(np.arange(l, l + m), 0, n - 1) - a]
        if lo1 is not None:
            out = crop(lo1, cnt1).copy()
            out[-cnt:] = crop(lo, cnt)
            r = end / out.shape[0]
            stash[c] = SlidingWindowFeature(out, SlidingWindow(start=0, duration=r, step=r))
        else:
            out = crop(lo, cnt)
            r = fixed / out.shape[0]
            stash[c] = SlidingWindowFeature(out, SlidingWindow(start=start, duration=r, step=r))
    return [stash.pop(c) for c in range(first, first + B)]


def _crop(data: np.ndarray, lo: int, cnt: int, n: int) -> np.ndarray:
    if lo >= 0 and lo + cnt <= n:
        return data[lo:lo + cnt]
    return data[np.clip(np.arange(lo, lo + cnt), 0, n - 1)]
