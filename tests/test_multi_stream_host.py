"""Host half of the multi-stream server (diart_b200/serve.py), without a GPU: the plan rows by chunk index, the window
bookkeeping of the slots and the per-stream time stamps."""
import types

import numpy as np
import pytest

from diart_b200.blocks.post import chunk_annotations, post_plan
from diart_b200.serve import MultiStreamDiarization, available_windows, plan_rows

SR, S, HOP, F = 16000, 80000, 8000, 293


def per_stream_plans(n, latency, step=0.5):
    """post_plan as SpeakerDiarization.__call__ runs it on a stream fed one window per call"""
    nw = int(round(latency / step))
    hist_s, hist_r, rows = np.zeros(0), np.zeros(0), []
    for i in range(n):
        start = i * step
        end = start + S * (1 / SR)
        res = (end - start if end > start else 0.0) / F
        plan, out_start, out_res = post_plan(np.array([start]), res, hist_s, hist_r, nw, F, step, latency)
        rows.append((plan[0], out_start[0], out_res[0]))
        keep = min(nw - 1, len(hist_s) + 1)
        hist_s = np.concatenate([hist_s, [start]])[len(hist_s) + 1 - keep:] if keep else np.zeros(0)
        hist_r = np.concatenate([hist_r, [res]])[len(hist_r) + 1 - keep:] if keep else np.zeros(0)
    return rows, nw


@pytest.mark.parametrize("latency", [0.5, 1.5, 2.0, 5.0])
def test_plan_rows_by_index_equal_post_plan_per_stream(latency):
    want, nw = per_stream_plans(120, latency)
    # the rows of a tick: several streams at different positions, grouped by stream
    idx = np.concatenate([np.arange(0, 4), np.arange(37, 40), np.arange(9, 10), np.arange(116, 120), np.arange(1, 3)])
    plan, out_start, out_res = plan_rows(idx, 0.5, S, SR, F, nw, latency)
    for r, i in enumerate(idx):
        assert np.array_equal(plan[r], want[i][0]), f"chunk {i}"
        assert out_start[r] == want[i][1] and out_res[r] == want[i][2], f"chunk {i}"
    # the first chunk of a stream emits the crop of [0, region end): at most F + 1 frames (dg_multi_step's bound)
    assert plan[0, 2] > 0 and plan[0, 2] <= F + 1


def test_available_windows_follow_ragged_pushes():
    rng = np.random.default_rng(3)
    pushed, emitted = np.zeros(5, np.int64), np.zeros(5, np.int64)
    ring = [np.zeros(0, np.float32) for _ in range(5)]     # everything each stream pushed
    for _ in range(60):
        for s in range(5):
            k = int(rng.integers(0, 30000))
            ring[s] = np.concatenate([ring[s], rng.standard_normal(k).astype(np.float32)])
            pushed[s] += k
        avail = available_windows(pushed, emitted, S, HOP)
        for s in range(5):
            # windows whose samples have all been pushed and that were not consumed
            n = 0
            while (emitted[s] + n) * HOP + S <= len(ring[s]):
                n += 1
            assert avail[s] == n
        emitted += np.minimum(avail, rng.integers(0, 5, size=5))


def test_window_start_times_carry_the_stream_shift():
    fake = types.SimpleNamespace(config=types.SimpleNamespace(step=0.5), _shift=np.array([0.0, 2.5]))
    assert MultiStreamDiarization.window_start_time(fake, 0, 7) == 3.5
    assert MultiStreamDiarization.window_start_time(fake, 1, 7) == 6.0


def test_per_chunk_shifts_give_the_scalar_shift_annotations():
    rng = np.random.default_rng(0)
    B, M = 6, 4
    counts = rng.integers(0, 3, size=B)
    header = np.zeros((B, 4), np.int32)
    header[:, 0] = np.cumsum(counts) - counts
    header[:, 1] = counts
    turns = np.array([(g << 20) | (on << 10) | (on + 5) for g, on in zip(rng.integers(0, M, counts.sum()),
                                                                           rng.integers(0, 200, counts.sum()))], np.uint32)
    out_start, out_res = rng.uniform(0, 30, B), np.full(B, 0.5 / 29)
    labels = [f"speaker{g}" for g in range(M)]
    shifts = np.array([0.0, 0.0, 3.25, 3.25, 1.5, 0.0])
    got = chunk_annotations(header, turns, len(turns), out_start, out_res, labels, shifts)
    for c in range(B):
        want = chunk_annotations(header, turns, len(turns), out_start, out_res, labels, float(shifts[c]))[c]
        assert got[c].to_rttm() == want.to_rttm() and got[c].modality == want.modality


def staging_run(slots, C, ops, samples):
    """dg_multi's bookkeeping of pushed audio through the host test hook -> (return codes, rings [slots][C])"""
    from diart_b200 import _lib
    ops = np.ascontiguousarray(np.asarray(ops, dtype=np.int32).reshape(-1, 3))
    samples = np.ascontiguousarray(samples, dtype=np.float32)
    result = np.zeros(len(ops), np.int32)
    rings = np.zeros((slots, C), np.float32)
    _lib.check(_lib.lib().dg_selftest_multi_staging_host(slots, C, len(ops), ops.ctypes.data, samples.ctypes.data,
                                                         result.ctypes.data, rings.ctypes.data))
    return result, rings


def staging_model(slots, C, ops, samples):
    """numpy model of the rings: a push is refused beyond C unconsumed samples, a close drops what the slot staged since the
    last tick, a tick writes every staged sample t of a slot at ring index t mod C"""
    is_open, wpos, rpos = [False] * slots, [0] * slots, [0] * slots
    pending = [[] for _ in range(slots)]
    rings = np.zeros((slots, C), np.float32)
    result, nxt = [], 0
    for kind, s, n in ops:
        rc = 0
        if kind == 0:
            rc = -1 if is_open[s] else 0
            if rc == 0:
                is_open[s], wpos[s], rpos[s] = True, 0, 0
        elif kind == 1:
            rc = 0 if is_open[s] else -1
            if rc == 0:
                is_open[s], pending[s] = False, []
        elif kind == 2:
            block = samples[nxt:nxt + n]
            nxt += n
            if not is_open[s] or wpos[s] + n - rpos[s] > C:
                rc = -1
            else:
                pending[s].append((wpos[s], block))
                wpos[s] += n
        elif kind == 3:
            rpos[s] += n
        else:
            for q in range(slots):
                for at, block in pending[q]:
                    rings[q, (at + np.arange(len(block))) % C] = block
                pending[q] = []
        result.append(rc)
    return np.array(result, np.int32), rings


def test_close_between_pushes_of_other_streams_drops_only_its_audio():
    """push(A), push(B), close(B), push(A) in one tick: A's two blocks land in A's ring, B's block nowhere"""
    ops = [(0, 0, 0), (0, 1, 0), (2, 0, 5), (2, 1, 7), (1, 1, 0), (2, 0, 6), (4, 0, 0)]
    samples = np.arange(1, 19, dtype=np.float32)
    got, want = staging_run(2, 64, ops, samples), staging_model(2, 64, ops, samples)
    assert np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1])
    assert np.array_equal(got[1][0, :11], np.r_[1:6, 13:19].astype(np.float32)) and not got[1][1].any()


def test_many_interleaved_small_pushes_pack_into_the_rings():
    """round-robin 20 ms frames of many streams (more pieces than a grid dimension holds), closes and reopens mid-tick,
    refused pushes, consumption and ring wrap-around, against the numpy model"""
    rng = np.random.default_rng(7)
    slots, C = 40, 4096
    ops, total = [(0, s, 0) for s in range(slots)], 0
    for tick in range(6):
        for _ in range(2000):
            s = int(rng.integers(0, slots))
            r = rng.random()
            if r < 0.02:
                ops += [(1, s, 0), (0, s, 0)]           # the stream ends and a new one takes its slot, mid-tick
            else:
                n = int(rng.integers(1, 320))
                ops.append((2, s, n))
                total += n
        ops.append((4, 0, 0))
        for s in range(slots):                          # a tick consumes some of what every slot holds
            ops.append((3, s, 0))
    # consumption amounts the model and the hook agree on: replay the model's counters
    samples = rng.standard_normal(total).astype(np.float32)
    wpos, rpos, final = np.zeros(slots, np.int64), np.zeros(slots, np.int64), []
    for kind, s, n in ops:
        if kind == 0:
            wpos[s] = rpos[s] = 0
        elif kind == 2 and wpos[s] + n - rpos[s] <= C:
            wpos[s] += n
        elif kind == 3:
            n = int((wpos[s] - rpos[s]) * 0.7)
            rpos[s] += n
        final.append((kind, s, n))
    got, want = staging_run(slots, C, final, samples), staging_model(slots, C, final, samples)
    assert np.array_equal(got[0], want[0])
    assert (want[0] == -1).any() and len(final) > 10000
    assert np.array_equal(got[1], want[1])
