"""Streams at other source rates in the multi-stream server, without a GPU: the tick's resampling plan (dg_multi's frame
items and window rows, through the host test hook) against a numpy model of the two rings of every slot, the plan rows on
a resampled stream's time base, and the rates the server refuses."""
import math
import types

import numpy as np
import pytest

from diart_b200.blocks.post import post_plan
from diart_b200.operators import sinc_resample_kernel
from diart_b200.serve import MultiStreamDiarization, plan_rows, source_geometry

SR, S, HOP, F = 16000, 80000, 8000, 293


def rate_row(rate, duration=5.0, step=0.5):
    """{o, n, w, chunk, step} of a source rate, as dg_multi_add_rate receives it"""
    g = math.gcd(rate, SR)
    _, w = sinc_resample_kernel(rate, SR)
    return [rate // g, SR // g, w, int(round(rate * duration)), int(round(rate * step))]


def frames_run(slots, max_wps, rates, ops, cap=1 << 20):
    from diart_b200 import _lib
    import ctypes as C
    r = np.ascontiguousarray(np.asarray(rates, dtype=np.int32).reshape(-1, 5))
    o = np.ascontiguousarray(np.asarray(ops, dtype=np.int32).reshape(-1, 3))
    result = np.zeros(len(o), np.int32)
    rec = np.zeros((cap, 5), np.int64)
    n = C.c_int()
    rc = _lib.lib().dg_selftest_multi_frames_host(slots, max_wps, S, HOP, len(r), r.ctypes.data, len(o), o.ctypes.data,
                                                  result.ctypes.data, rec.ctypes.data, cap, C.byref(n))
    return rc, result, rec[:n.value]


class Geom:
    def __init__(self, row, max_wps):
        if row is None:                                        # the pipeline's rate
            self.o, self.S, self.hop = 0, S, HOP
        else:
            self.o, self.n, self.w, self.S, self.hop = row
            self.T = 2 * self.w + self.o
            self.fs = self.hop // self.o
            self.r_lo = -(-self.w // self.o)
            self.r_hi = (self.S - self.w - self.o) // self.o
            self.Q = (max_wps - 1) * self.fs + self.r_hi - self.r_lo + 1
        self.cap = -(-(self.S + 2 * max_wps * self.hop) // 1024) * 1024


def check_against_model(slots, max_wps, rate_rows, ops):
    """runs the hook and replays ops on a model of every slot: samples pushed / consumed, and its 16 kHz ring as
    physical storage tagged (stream generation, frame) -- it is NOT cleared when the slot is reopened"""
    rc, result, rec = frames_run(slots, max_wps, rate_rows, ops)
    assert rc == 0
    geoms = [Geom(None, max_wps)] + [Geom(r, max_wps) for r in rate_rows]
    max_q = max([g.Q for g in geoms[1:]] + [1])
    is_open, rate = [False] * slots, [0] * slots
    wpos, rpos, gen = [0] * slots, [0] * slots, [0] * slots
    computed = [set() for _ in range(slots)]
    ring16 = [[None] * max_q for _ in range(slots)]
    tick, stats = 0, dict(items=0, windows=0, wrap_src=False, wrap16=False, reopened_other_rate=False)
    for i, (kind, s, n) in enumerate(ops):
        want_rc = 0
        if kind == 0:
            if is_open[s] or not -1 <= n < len(rate_rows):
                want_rc = -1
            else:
                stats["reopened_other_rate"] |= gen[s] > 0 and rate[s] != n + 1
                is_open[s], rate[s], wpos[s], rpos[s] = True, n + 1, 0, 0
                gen[s] += 1
                computed[s] = set()
        elif kind == 1:
            want_rc = 0 if is_open[s] else -1
            is_open[s] = False
        elif kind == 2:
            if not is_open[s] or wpos[s] + n - rpos[s] > geoms[rate[s]].cap:
                want_rc = -1
            else:
                wpos[s] += n
        else:
            mine = rec[rec[:, 0] == tick]
            items, rows = mine[mine[:, 1] == 0], mine[mine[:, 1] == 1]
            # the windows: every open slot in slot order, min(available, max_wps) each, consecutive batch rows
            want_rows, b = [], 0
            for q in range(slots):
                g = geoms[rate[q]]
                have = wpos[q] - rpos[q]
                k = 0 if not is_open[q] or have < g.S else min((have - g.S) // g.hop + 1, max_wps)
                want_rows += [(q, rpos[q] + j * g.hop, b + j) for j in range(k)]
                b += k
            assert [tuple(r[2:]) for r in rows] == want_rows, f"tick {tick}: window rows"
            # the items: frames never computed before, every tap pushed and still in the source ring
            for _, _, q, first, count in items:
                g = geoms[rate[q]]
                assert g.o, f"tick {tick}: a resampling item for slot {q} at the pipeline's rate"
                for R in range(first, first + count):
                    assert R not in computed[q], f"tick {tick}: frame {R} of slot {q} computed twice"
                    assert R * g.o - g.w >= max(rpos[q], wpos[q] - g.cap), f"tick {tick}: frame {R} needs a dropped sample"
                    assert R * g.o - g.w + g.T <= wpos[q], f"tick {tick}: frame {R} needs a sample not pushed"
                    computed[q].add(R)
                    stats["wrap16"] |= R >= g.Q
                    ring16[q][R % g.Q] = (gen[q], R)
                stats["items"] += 1
            # every interior frame of every window is in the 16 kHz ring, from this stream
            for q, start, _ in want_rows:
                g = geoms[rate[q]]
                if g.o:
                    f0 = start // g.o
                    assert start % g.o == 0
                    for r in range(g.r_lo, g.r_hi + 1):
                        assert ring16[q][(f0 + r) % g.Q] == (gen[q], f0 + r), f"tick {tick}: slot {q} frame {f0 + r}"
                stats["wrap_src"] |= start + g.S > g.cap
                rpos[q] += g.hop
                stats["windows"] += 1
            # frames computed are one run from the first window's first interior frame
            for q in range(slots):
                if is_open[q] and geoms[rate[q]].o and computed[q]:
                    g = geoms[rate[q]]
                    assert computed[q] == set(range(g.r_lo, max(computed[q]) + 1))
            tick += 1
        assert result[i] == want_rc, f"op {i} {kind, s, n}"
    return stats, result, rec


def ragged_ops(rng, slots, rate_of, geoms, ticks, max_wps, reopen=None):
    """per tick, each open slot pushes 0 .. max_wps + 1 hops' worth in ragged blocks: shorter than a hop, or longer
    than a window (some beyond the ring capacity: refused)"""
    ops = [(0, s, rate_of[s]) for s in range(slots)]
    for t in range(ticks):
        for s in range(slots):
            g = geoms[rate_of[s] + 1]
            target = int(rng.integers(0, max_wps + 2)) * g.hop
            while target > 0:
                k = int(rng.integers(1, g.hop)) if rng.random() < 0.7 else int(rng.integers(g.S + 1, g.S + 2 * g.hop))
                ops.append((2, s, k))
                target -= k
            if reopen and t == reopen[0] and s == 0:
                # slot reopen[1] ends between two pushes of stream 0, a new stream at another rate takes it
                ops += [(1, reopen[1], 0), (2, 0, 77), (0, reopen[1], reopen[2])]
                rate_of[reopen[1]] = reopen[2]
        ops.append((4, 0, 0))
    return ops


def test_frame_plan_against_the_ring_model():
    rates = [44100, 48000, 22050]
    rows = [rate_row(r) for r in rates]
    max_wps = 4
    geoms = [Geom(None, max_wps)] + [Geom(r, max_wps) for r in rows]
    rng = np.random.default_rng(5)
    rate_of = [-1, 0, 1, 2, 0, 2]
    ops = ragged_ops(rng, 6, list(rate_of), geoms, 60, max_wps, reopen=(23, 1, 1))
    stats, result, rec = check_against_model(6, max_wps, rows, ops)
    assert stats["wrap_src"] and stats["wrap16"] and stats["reopened_other_rate"]
    assert (result == -1).any(), "no push beyond a ring's capacity was tried"
    rows_of = rec[rec[:, 1] == 1]
    per_slot_tick = np.zeros((60, 6), np.int64)
    np.add.at(per_slot_tick, (rows_of[:, 0], rows_of[:, 2]), 1)
    assert set(np.unique(per_slot_tick)) == set(range(max_wps + 1)), "0 to max_wps windows per stream and tick"
    assert stats["items"] > 100 and stats["windows"] > 300


@pytest.mark.parametrize("max_wps", [1, 2])
def test_frame_plan_one_window_per_tick(max_wps):
    """a hop per tick: each tick computes fs new frames per stream, after a first tick of a window's interior
    (issue geometry: 44.1 kHz 1 .. 498, 48 kHz 7 .. 79 992, 22.05 kHz 1 .. 248)"""
    rows = [rate_row(r) for r in (44100, 48000, 22050)]
    ops = [(0, s, s) for s in range(3)] + [(0, 3, -1)]
    for t in range(30):
        for s in range(4):
            g = Geom(rows[s] if s < 3 else None, max_wps)
            ops.append((2, s, g.S if t == 0 else g.hop))
        ops.append((4, 0, 0))
    stats, _, rec = check_against_model(4, max_wps, rows, ops)
    items = rec[rec[:, 1] == 0]
    first = {int(s): (int(a), int(b)) for _, _, s, a, b in items[items[:, 0] == 0]}
    assert first == {0: (1, 498), 1: (7, 79986), 2: (1, 248)}
    later = items[items[:, 0] == 5]
    assert [int(b) for b in later[:, 4]] == [50, 8000, 25]
    assert stats["wrap16"]


def test_frame_plan_refusals():
    row = rate_row(44100)
    bad_chunk = row[:3] + [row[3] + 1, row[4]]                 # resamples to 80 001 samples
    bad_step = row[:3] + [row[3], int(round(44100 * 0.125))]   # 5 512 samples: not whole frames of 441
    for rates in ([bad_chunk], [bad_step]):
        rc, _, _ = frames_run(2, 4, rates, [(0, 0, -1)])
        assert rc == -1
    # opening at a rate id that was not declared
    rc, result, _ = frames_run(2, 4, [row], [(0, 0, 1), (0, 0, 0), (0, 1, -1), (0, 1, 0)])
    assert rc == 0 and list(result) == [-1, 0, 0, -1]


def test_source_geometry_refusals():
    assert source_geometry(44100, SR, 5.0, 0.5) == (220500, 22050, (220500 * (1 / 44100)) / 80000)
    for rate in (8000, 22050, 32000, 44100, 48000):
        source_geometry(rate, SR, 5.0, 0.5)
    with pytest.raises(ValueError):
        source_geometry(44100, SR, 5.0, 0.125)                 # step % o != 0
    with pytest.raises(ValueError):
        source_geometry(44100, SR, 5.00002, 0.5)               # the chunk resamples to 80 001 samples
    fake = types.SimpleNamespace(config=types.SimpleNamespace(sample_rate=SR), rates={SR: (-1, S, HOP, 1 / SR)},
                                 _resamplers={})
    with pytest.raises(ValueError):
        MultiStreamDiarization.open(fake, 0.0, 44100)          # a rate that was not declared


def per_stream_plans(n, latency, res, step=0.5):
    """post_plan as SpeakerDiarization.__call__ runs it on a stream of windows of S samples spaced `res` apart, one per call"""
    nw = int(round(latency / step))
    hist_s, hist_r, rows = np.zeros(0), np.zeros(0), []
    for i in range(n):
        start = i * step
        end = start + S * res
        r = (end - start if end > start else 0.0) / F
        plan, out_start, out_res = post_plan(np.array([start]), r, hist_s, hist_r, nw, F, step, latency)
        rows.append((plan[0], out_start[0], out_res[0]))
        keep = min(nw - 1, len(hist_s) + 1)
        hist_s = np.concatenate([hist_s, [start]])[len(hist_s) + 1 - keep:] if keep else np.zeros(0)
        hist_r = np.concatenate([hist_r, [r]])[len(hist_r) + 1 - keep:] if keep else np.zeros(0)
    return rows, nw


@pytest.mark.parametrize("latency", [0.5, 2.0, 5.0])
def test_plan_rows_per_rate_equal_post_plan_per_stream(latency):
    res = {r: source_geometry(r, SR, 5.0, 0.5)[2] for r in (16000, 44100, 48000, 22050)}
    want = {r: per_stream_plans(60, latency, res[r]) for r in res}
    nw = want[16000][1]
    # a tick's rows: streams at several rates and positions, grouped by stream
    parts = [(44100, np.arange(0, 4)), (16000, np.arange(37, 40)), (48000, np.arange(9, 10)), (22050, np.arange(56, 60)),
             (16000, np.arange(1, 3)), (44100, np.arange(20, 22))]
    idx = np.concatenate([p for _, p in parts])
    rates = np.concatenate([[r] * len(p) for r, p in parts])
    plan, out_start, out_res = plan_rows(idx, 0.5, S, SR, F, nw, latency, np.array([res[r] for r in rates]))
    for row, (i, r) in enumerate(zip(idx, rates)):
        w = want[r][0][i]
        assert np.array_equal(plan[row], w[0]) and out_start[row] == w[1] and out_res[row] == w[2], f"{r} Hz chunk {i}"
    # rows at the pipeline's rate come out as they do without a resolution
    plain = plan_rows(idx, 0.5, S, SR, F, nw, latency)
    at16 = rates == 16000
    for a, b in zip(plain, (plan, out_start, out_res)):
        assert np.array_equal(a[at16], b[at16])
