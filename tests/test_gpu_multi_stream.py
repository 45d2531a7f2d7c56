"""Many live streams on one device (diart_b200.serve.MultiStreamDiarization, dg_multi_*): every stream gets exactly what a
dedicated SpeakerDiarization gives on its windows fed one per call (the reference's live mode), whatever the other streams
do in the same ticks.

Scores, speaker maps and RTTM are compared bit for bit.  Embeddings are compared within EMB_TOL: the fused TDNN5 pooling adds
per-tile partial sums whose split follows the window's row offset in the batch, so a window's embedding can differ in the
last bits between batch positions (the single-stream pipeline has the same property; only scores are batch invariant)."""
import ctypes as C

import numpy as np
import pytest
import torch

from diart_b200 import _lib, blocks, models, synth
from diart_b200.core import SlidingWindow, SlidingWindowFeature
from diart_b200.serve import MultiStreamDiarization

pytestmark = pytest.mark.gpu

SR, S, HOP = 16000, 80000, 8000
EMB_TOL = 1e-5


def make_config(oracle_nets, device, **kw):
    seg_o, emb_o = oracle_nets
    return blocks.SpeakerDiarizationConfig(
        segmentation=models.SegmentationModel(models.B200SegmentationLoader(seg_o.state_dict())),
        embedding=models.EmbeddingModel(models.B200EmbeddingLoader(emb_o.state_dict())), device=device, **kw)


def window(audio, i):
    return SlidingWindowFeature(audio[i * HOP:i * HOP + S, None], SlidingWindow(start=i * 0.5, duration=1 / SR, step=1 / SR))


def dedicated(config, audio, n, shift=0.0):
    """the reference's live mode: a SpeakerDiarization per stream, one window per call -> (RTTM per window, and the scores,
    embeddings and maps of each window's fused step from a second pipeline in the same state)"""
    pipe, twin = blocks.SpeakerDiarization(config), blocks.SpeakerDiarization(config)
    pipe.set_timestamp_shift(shift)
    rttm, seg, emb, maps = [], [], [], []
    for i in range(n):
        rttm.append(pipe([window(audio, i)])[0][0].to_rttm())
        s, e, m = twin.device_step(torch.from_numpy(synth.windows(audio, 1, first=i)).to(config.device))
        seg.append(s.cpu().numpy()[0]), emb.append(e.cpu().numpy()[0]), maps.append(m.cpu().numpy()[0])
    return rttm, np.stack(seg), np.stack(emb), np.stack(maps)


class Recorder:
    """runs ticks of a server and keeps, per stream key, its annotations and its rows of the tick outputs"""

    def __init__(self, server):
        self.server, self.rttm, self.seg, self.emb, self.maps = server, {}, {}, {}, {}
        self.sid_key = {}

    def tick(self):
        res, outs = self.server._step(outputs=True)
        sids = sorted(res)
        if outs is not None:
            seg, emb, maps = (t.cpu().numpy() for t in outs)
        r = 0
        for sid in sids:
            key, n = self.sid_key[sid], len(res[sid])
            self.rttm.setdefault(key, []).extend(a.to_rttm() for a in res[sid])
            for store, arr in ((self.seg, seg), (self.emb, emb), (self.maps, maps)):
                store.setdefault(key, []).extend(arr[r:r + n])
            r += n
        return sum(len(v) for v in res.values())


@pytest.mark.parametrize("kw", [dict(latency=0.5), dict(latency=2.0), dict(latency=2.0, max_speakers=4)],
                         ids=["latency0.5", "latency2", "speakers4"])
def test_streams_equal_dedicated_pipelines(oracle_nets, cuda_device, kw):
    config = make_config(oracle_nets, cuda_device, **kw)
    rng = np.random.default_rng(11)
    # (seed, windows, tick at which the stream opens, timestamp shift); stream 1 is closed after 9 windows and stream 6
    # then opens in its slot
    plan = [(101, 40, 0, 0.0), (102, 70, 0, 0.0), (103, 33, 2, 3.25), (104, 45, 5, 0.0), (105, 20, 1, 0.0), (106, 52, 3, 0.0),
            (107, 24, None, 1.5)]
    audio = {k: synth.synth_audio(S + HOP * (n - 1), seed=seed) for k, (seed, n, _, _) in enumerate(plan)}
    want = {k: dedicated(config, audio[k], 9 if k == 1 else n, shift) for k, (_, n, _, shift) in enumerate(plan)}
    server = MultiStreamDiarization(config, max_streams=6, max_windows_per_stream=4)
    rec = Recorder(server)
    pos, sid_of, done = {}, {}, set()
    per_tick, tick = [], 0
    while len(done) < len(plan):
        for k, (_, n, t_open, shift) in enumerate(plan):
            if k not in sid_of and k not in done and (t_open == tick or (k == 6 and 1 in done)):
                sid_of[k] = server.open(shift)
                rec.sid_key[sid_of[k]] = k
                pos[k] = 0
                if k == 6:
                    assert sid_of[k] == sid_of_closed, "the new stream takes the closed stream's slot"
        for k, sid in list(sid_of.items()):
            a = audio[k]
            room = server.window_samples + 2 * 4 * HOP - (server._pushed[sid] - server._emitted[sid] * HOP)
            # ragged blocks: shorter than a hop, or longer than a window
            size = int(rng.integers(500, HOP)) if rng.random() < 0.6 else int(rng.integers(S + 1, S + 30000))
            size = min(size, room, len(a) - pos[k])
            if size > 0:
                server.push(sid, a[pos[k]:pos[k] + size][None, :] if rng.random() < 0.5 else a[pos[k]:pos[k] + size])
                pos[k] += size
        per_tick.append(rec.tick())
        tick += 1
        for k, sid in list(sid_of.items()):
            got = len(rec.rttm.get(k, []))
            if (k == 1 and got >= 9) or got == plan[k][1]:
                server.close(sid)
                del sid_of[k]
                done.add(k)
                if k == 1:
                    sid_of_closed = sid
        assert tick < 200
    assert 0 in per_tick and max(per_tick) > 6, per_tick
    for k, (rttm, seg, emb, maps) in want.items():
        n = len(rttm)
        assert rec.rttm[k][:n] == rttm, f"stream {k}: RTTM differs"
        assert np.array_equal(np.stack(rec.seg[k][:n]), seg), f"stream {k}: scores differ"
        assert np.abs(np.stack(rec.emb[k][:n]) - emb).max() <= EMB_TOL, f"stream {k}: embeddings differ"
        assert np.array_equal(np.stack(rec.maps[k][:n]), maps), f"stream {k}: speaker maps differ"


def run_streams(server, audios, ticks):
    """every stream pushes its first window, then one hop per tick"""
    rec = Recorder(server)
    for k in range(len(audios)):
        rec.sid_key[server.open()] = k
    for t in range(ticks):
        for sid, k in rec.sid_key.items():
            a = audios[k]
            server.push(sid, a[:S] if t == 0 else a[S + (t - 1) * HOP:S + t * HOP])
        rec.tick()
    return rec


def test_a_stream_alone_equals_it_among_300(oracle_nets, cuda_device):
    """300 windows per tick: two network sub-batches, and more clustering states than one wave of CTAs.  Stream 137 sits at
    batch row 137 among 300, at row 0 alone"""
    config = make_config(oracle_nets, cuda_device, latency=2.0)
    ticks = 5
    base = [synth.synth_audio(S + HOP * (ticks - 1) + 40 * HOP, seed=300 + i) for i in range(6)]
    audios = [np.ascontiguousarray(base[i % 6][(i // 6) % 40 * HOP:][:S + HOP * (ticks - 1)]) for i in range(300)]
    alone = run_streams(MultiStreamDiarization(config, max_streams=1, max_windows_per_stream=1), [audios[137]], ticks)
    crowd = run_streams(MultiStreamDiarization(config, max_streams=300, max_windows_per_stream=1), audios, ticks)
    assert len(crowd.rttm[137]) == ticks
    assert crowd.rttm[137] == alone.rttm[0]
    for store_c, store_a in ((crowd.seg, alone.seg), (crowd.maps, alone.maps)):
        assert np.array_equal(np.stack(store_c[137]), np.stack(store_a[0]))
    assert np.abs(np.stack(crowd.emb[137]) - np.stack(alone.emb[0])).max() <= EMB_TOL


def test_shared_models_interleaved(oracle_nets, cuda_device):
    """a SpeakerDiarization and a server on the same model objects, calls interleaved: each gives its solo results"""
    config = make_config(oracle_nets, cuda_device, latency=1.5)
    n = 12
    a_pipe, a_srv = synth.synth_audio(S + HOP * (n - 1), seed=71), synth.synth_audio(S + HOP * (n - 1), seed=72)
    alone = blocks.SpeakerDiarization(config)
    solo_pipe = [alone([window(a_pipe, i)])[0][0].to_rttm() for i in range(n)]
    solo_srv = run_streams(MultiStreamDiarization(config, 2), [a_srv], n).rttm[0]
    pipe, server = blocks.SpeakerDiarization(config), MultiStreamDiarization(config, 2)
    sid = server.open()
    got_pipe, got_srv = [], []
    for i in range(n):
        server.push(sid, a_srv[:S] if i == 0 else a_srv[S + (i - 1) * HOP:S + i * HOP])
        got_srv += [a.to_rttm() for a in server.step()[sid]]
        got_pipe.append(pipe([window(a_pipe, i)])[0][0].to_rttm())
    assert got_pipe == solo_pipe and got_srv == solo_srv


def test_refusals(oracle_nets, cuda_device):
    config = make_config(oracle_nets, cuda_device)
    server = MultiStreamDiarization(config, max_streams=2, max_windows_per_stream=2)
    lib = _lib.lib()
    a = synth.synth_audio(S + 4 * HOP, seed=5)
    sid = server.open()
    server.push(sid, a[:S + HOP])
    assert server.available(sid) == 2
    with pytest.raises(ValueError):                     # more than the ring holds: refused, nothing written
        server.push(sid, np.zeros(S + 4 * HOP, np.float32))
    assert server.available(sid) == 2
    with pytest.raises(ValueError):                     # unknown slot
        server.push(7, a[:10])
    other = server.open()
    with pytest.raises(ValueError):                     # more than max_streams open
        server.open()
    assert lib.dg_multi_open(server.handle, 2) == _lib.lib().dg_multi_open(server.handle, -1) == -1
    server.close(other)
    with pytest.raises(ValueError):                     # closed slot
        server.push(other, a[:10])
    with pytest.raises(ValueError):
        server.available(other)
    counts, header, turns, nt = np.empty(2, np.int32), np.empty((4, 4), np.int32), np.empty(64, np.uint32), C.c_int()
    plan = np.zeros((4, 4 + server.nw), np.int32)
    # a plan for another number of windows than the tick has
    assert lib.dg_multi_step(server.handle, plan.ctypes.data, 1, counts.ctypes.data, header.ctypes.data, turns.ctypes.data,
                             64, C.byref(nt), None, None, None) == -1
    # the refused push wrote nothing: the windows are those of the audio
    got = server.step()[sid]
    pipe = blocks.SpeakerDiarization(config)
    assert [g.to_rttm() for g in got] == [pipe([window(a, i)])[0][0].to_rttm() for i in range(2)]
    # a tick with nothing available launches nothing
    before = lib.dg_launch_count()
    assert server.step() == {}
    assert lib.dg_launch_count() == before


def test_small_frames_and_a_close_inside_a_tick(oracle_nets, cuda_device):
    """300 streams push 20 ms frames round robin (about 75 000 staged pieces in the first tick, more than a grid dimension
    holds); inside that tick stream 1 is closed between two pushes of stream 0, and a new stream takes slot 1 and catches up.
    Streams 0 and 2 and the new stream equal their dedicated pipelines"""
    config = make_config(oracle_nets, cuda_device)
    ticks, frame = 4, 320
    base = [synth.synth_audio(S + HOP * (ticks - 1) + 40 * HOP, seed=500 + i) for i in range(6)]
    audios = [np.ascontiguousarray(base[i % 6][(i // 6) % 40 * HOP:][:S + HOP * (ticks - 1)]) for i in range(300)]
    audios.append(synth.synth_audio(S + HOP * (ticks - 1), seed=599))            # the stream that reuses slot 1
    server = MultiStreamDiarization(config, max_streams=300, max_windows_per_stream=1)
    rec = Recorder(server)
    key_of = {}
    for k in range(300):
        key_of[k] = server.open()
        rec.sid_key[key_of[k]] = k
    pushed = {k: 0 for k in key_of}

    def push_frame(k):
        n = min(frame, target - pushed[k])
        server.push(key_of[k], audios[k][pushed[k]:pushed[k] + n])
        pushed[k] += n

    for t in range(ticks):
        target = S + t * HOP
        rounds = 0
        while any(pushed[k] < target for k in key_of):
            for k in list(key_of):
                if pushed[k] < target:
                    push_frame(k)
                if t == 0 and rounds == 100 and k == 1:
                    server.close(key_of.pop(1))
                    key_of[300] = server.open()
                    assert key_of[300] == 1
                    rec.sid_key[1] = 300
                    pushed[300] = 0
                    push_frame(0)                         # stream 0 continues right after the close
            rounds += 1
        rec.tick()
    for k in (0, 2, 300):
        n = len(rec.rttm[k])
        assert n == ticks
        rttm, seg, emb, maps = dedicated(config, audios[k], n)
        assert rec.rttm[k] == rttm, f"stream {k}: RTTM differs"
        assert np.array_equal(np.stack(rec.seg[k]), seg), f"stream {k}: scores differ"
        assert np.array_equal(np.stack(rec.maps[k]), maps), f"stream {k}: speaker maps differ"
        assert np.abs(np.stack(rec.emb[k]) - emb).max() <= EMB_TOL, f"stream {k}: embeddings differ"
