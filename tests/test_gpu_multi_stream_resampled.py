"""Streams at 22.05, 44.1 and 48 kHz in the multi-stream server (MultiStreamDiarization(source_sample_rates=...),
dg_multi_add_rate): every resampled window of a tick has the bits of DeviceResample on the stacked source windows, and every
stream gets exactly what a dedicated SpeakerDiarization gives on its resampled windows fed one per call.

Scores, speaker maps and RTTM are compared bit for bit; embeddings within EMB_TOL, for the reason test_gpu_multi_stream.py
gives (the fused TDNN5 pooling's partial sums follow a window's row in the batch)."""
import ctypes as C

import numpy as np
import pytest
import torch

from diart_b200 import _lib, blocks, synth
from diart_b200.core import SlidingWindow, SlidingWindowFeature
from diart_b200.operators import DeviceResample
from diart_b200.serve import MultiStreamDiarization, source_geometry
from test_gpu_multi_stream import EMB_TOL, Recorder, make_config

pytestmark = pytest.mark.gpu

SR, S = 16000, 80000
RATES = (44100, 48000, 22050)


def source(n_windows, rate, seed):
    chunk, hop, _ = source_geometry(rate, SR, 5.0, 0.5)
    return synth.synth_audio(chunk + hop * (n_windows - 1), seed=seed, sample_rate=rate)


def stacked(audio, rate, first, n):
    chunk, hop, _ = source_geometry(rate, SR, 5.0, 0.5)
    return np.stack([audio[(first + i) * hop:(first + i) * hop + chunk] for i in range(n)])


class Windows:
    """the reference's windows of a stream at `rate`: rearrange_audio_stream at that rate, then Resample (DeviceResample)"""

    def __init__(self, device):
        self.rs = {r: DeviceResample(r, SR, device) for r in RATES}
        self.device = device

    def __call__(self, audio, rate, first, n):
        x = torch.from_numpy(np.ascontiguousarray(stacked(audio, rate, first, n))).to(self.device)
        return (self.rs[rate](x) if rate != SR else x).cpu().numpy()


def last_windows(server, B):
    out = torch.empty((B, S), device=server.device)
    _lib.check(_lib.lib().dg_multi_last_windows(server.handle, out.data_ptr(), B))
    return out.cpu().numpy()


def test_tick_windows_equal_resampled_stacked_windows(oracle_nets, cuda_device):
    """16, 44.1, 48 and 22.05 kHz streams in the same ticks, ragged pushes (shorter than a hop, longer than a window), up to
    4 windows per stream and tick, both rings of every slot wrapping around, a slot reopened at another rate"""
    config = make_config(oracle_nets, cuda_device)
    server = MultiStreamDiarization(config, max_streams=6, max_windows_per_stream=4, source_sample_rates=RATES)
    ref = Windows(cuda_device)
    rng = np.random.default_rng(3)
    plan = [SR, 44100, 48000, 22050, 44100, 48000]
    n_win = 36
    audio = {k: source(n_win, r, 200 + k) for k, r in enumerate(plan)}
    sid = {k: server.open(sample_rate=r) for k, r in enumerate(plan)}
    pos = {k: 0 for k in sid}
    checked = {k: 0 for k in sid}
    reopened = False
    for tick in range(200):
        for k in list(sid):
            chunk, hop, _ = source_geometry(plan[k], SR, 5.0, 0.5)
            room = chunk + 8 * hop - (server._pushed[sid[k]] - server._emitted[sid[k]] * hop)
            size = int(rng.integers(100, hop)) if rng.random() < 0.6 else int(rng.integers(chunk + 1, chunk + 3 * hop))
            size = min(size, room, len(audio[k]) - pos[k])
            if size > 0:
                server.push(sid[k], audio[k][pos[k]:pos[k] + size])
                pos[k] += size
        before = server._emitted.copy()
        res = server.step()
        B = sum(len(v) for v in res.values())
        if B:
            got = last_windows(server, B)
            r0 = 0
            for s in sorted(res):
                k = next(k for k, v in sid.items() if v == s)
                n = len(res[s])
                want = ref(audio[k], plan[k], int(before[s]), n)
                assert np.array_equal(got[r0:r0 + n].view(np.uint32), want.view(np.uint32)), \
                    f"tick {tick}: stream {k} at {plan[k]} Hz, windows {before[s]} .. {before[s] + n}"
                checked[k] += n
                r0 += n
        if not reopened and checked[1] >= 12:
            # stream 1 (44.1 kHz) ends; a 22.05 kHz stream takes its slot
            server.close(sid[1])
            plan[1] = 22050
            audio[1] = source(n_win, 22050, 299)
            sid[1], pos[1], checked[1] = server.open(sample_rate=22050), 0, 0
            reopened = True
        if all(checked[k] >= n_win for k in sid):
            break
    assert reopened and all(checked[k] >= n_win for k in sid), checked


def dedicated(config, x, shift=0.0, res=1 / SR):
    """the reference's live mode on resampled windows x (n, S): a SpeakerDiarization, one window per call (RTTM), and the
    scores, embeddings and maps of each window's fused step from a second pipeline in the same state"""
    pipe, twin = blocks.SpeakerDiarization(config), blocks.SpeakerDiarization(config)
    pipe.set_timestamp_shift(shift)
    rttm, seg, emb, maps = [], [], [], []
    for i in range(len(x)):
        w = SlidingWindowFeature(x[i, :, None], SlidingWindow(start=i * 0.5, duration=res, step=res))
        rttm.append(pipe([w])[0][0].to_rttm())
        s, e, m = twin.device_step(torch.from_numpy(x[i:i + 1]).to(config.device))
        seg.append(s.cpu().numpy()[0]), emb.append(e.cpu().numpy()[0]), maps.append(m.cpu().numpy()[0])
    return rttm, np.stack(seg), np.stack(emb), np.stack(maps)


def assert_same(rec, k, want):
    rttm, seg, emb, maps = want
    n = len(rttm)
    assert rec.rttm[k][:n] == rttm, f"stream {k}: RTTM differs"
    assert np.array_equal(np.stack(rec.seg[k][:n]), seg), f"stream {k}: scores differ"
    assert np.abs(np.stack(rec.emb[k][:n]) - emb).max() <= EMB_TOL, f"stream {k}: embeddings differ"
    assert np.array_equal(np.stack(rec.maps[k][:n]), maps), f"stream {k}: speaker maps differ"


@pytest.mark.parametrize("kw", [dict(latency=0.5), dict(latency=2.0), dict(latency=2.0, max_speakers=4)],
                         ids=["latency0.5", "latency2", "speakers4"])
def test_streams_equal_dedicated_pipelines_on_resampled_windows(oracle_nets, cuda_device, kw):
    config = make_config(oracle_nets, cuda_device, **kw)
    ref = Windows(cuda_device)
    rng = np.random.default_rng(17)
    # (rate, windows, timestamp shift)
    plan = [(44100, 14, 0.0), (SR, 12, 1.5), (48000, 13, 3.25), (22050, 14, 0.0), (44100, 11, 2.0)]
    audio = {k: source(n, r, 400 + k) for k, (r, n, _) in enumerate(plan)}
    server = MultiStreamDiarization(config, max_streams=len(plan), max_windows_per_stream=4, source_sample_rates=RATES)
    rec = Recorder(server)
    sid = {}
    for k, (r, _, shift) in enumerate(plan):
        sid[k] = server.open(shift=shift, sample_rate=r)
        rec.sid_key[sid[k]] = k
    pos = {k: 0 for k in sid}
    for _ in range(100):
        for k, (r, _, _) in enumerate(plan):
            chunk, hop, _ = source_geometry(r, SR, 5.0, 0.5)
            room = chunk + 8 * hop - (server._pushed[sid[k]] - server._emitted[sid[k]] * hop)
            size = int(rng.integers(300, hop)) if rng.random() < 0.6 else int(rng.integers(chunk + 1, chunk + 2 * hop))
            size = min(size, room, len(audio[k]) - pos[k])
            if size > 0:
                server.push(sid[k], audio[k][pos[k]:pos[k] + size])
                pos[k] += size
        rec.tick()
        if all(len(rec.rttm.get(k, [])) == n for k, (_, n, _) in enumerate(plan)):
            break
    for k, (r, n, shift) in enumerate(plan):
        assert len(rec.rttm[k]) == n
        assert_same(rec, k, dedicated(config, ref(audio[k], r, 0, n), shift, source_geometry(r, SR, 5.0, 0.5)[2]))


def run_streams(server, audios, rates, ticks):
    """every stream pushes its first window, then one hop per tick"""
    rec = Recorder(server)
    for k, r in enumerate(rates):
        rec.sid_key[server.open(sample_rate=r)] = k
    for t in range(ticks):
        for sid, k in rec.sid_key.items():
            chunk, hop, _ = source_geometry(rates[k], SR, 5.0, 0.5)
            a = audios[k]
            server.push(sid, a[:chunk] if t == 0 else a[chunk + (t - 1) * hop:chunk + t * hop])
        rec.tick()
    return rec


def test_a_resampled_stream_alone_equals_it_among_300(oracle_nets, cuda_device):
    """300 streams at 16, 44.1, 48 and 22.05 kHz: two network sub-batches and many resampling items per launch.  Stream 137
    (44.1 kHz) sits at batch row 137 among 300, at row 0 alone"""
    config = make_config(oracle_nets, cuda_device, latency=2.0)
    ticks = 4
    mix = (SR, 44100, 48000, 22050)
    rates = [mix[i % 4] for i in range(300)]
    base = {r: [source(ticks + 30, r, 600 + 10 * j + r % 7) for j in range(3)] for r in mix}

    def cut(i):
        chunk, hop, _ = source_geometry(rates[i], SR, 5.0, 0.5)
        return np.ascontiguousarray(base[rates[i]][i % 3][(i // 4) % 30 * hop:][:chunk + hop * (ticks - 1)])

    audios = [cut(i) for i in range(300)]
    assert rates[137] == 44100
    alone = run_streams(MultiStreamDiarization(config, 1, 1, source_sample_rates=RATES), [audios[137]], [44100], ticks)
    crowd = run_streams(MultiStreamDiarization(config, 300, 1, source_sample_rates=RATES), audios, rates, ticks)
    assert len(crowd.rttm[137]) == ticks and crowd.rttm[137] == alone.rttm[0]
    for store_c, store_a in ((crowd.seg, alone.seg), (crowd.maps, alone.maps)):
        assert np.array_equal(np.stack(store_c[137]), np.stack(store_a[0]))
    assert np.abs(np.stack(crowd.emb[137]) - np.stack(alone.emb[0])).max() <= EMB_TOL


def test_16khz_ticks_unchanged_by_declared_rates(oracle_nets, cuda_device):
    """16 kHz streams only: the same launches and the same bits with and without declared rates"""
    config = make_config(oracle_nets, cuda_device, latency=1.5)
    ticks, n = 4, 5
    audios = [source(ticks, SR, 700 + i) for i in range(n)]
    lib = _lib.lib()
    recs, launches = [], []
    for rates in ((), RATES):
        server = MultiStreamDiarization(config, max_streams=n, max_windows_per_stream=2, source_sample_rates=rates)
        rec = Recorder(server)
        for k in range(n):
            rec.sid_key[server.open()] = k
        counts = []
        for t in range(ticks):
            for sid, k in rec.sid_key.items():
                server.push(sid, audios[k][:S] if t == 0 else audios[k][S + (t - 1) * 8000:S + t * 8000])
            before = lib.dg_launch_count()
            res = server.step()
            counts.append(lib.dg_launch_count() - before)
            for s, anns in res.items():
                rec.rttm.setdefault(rec.sid_key[s], []).extend(a.to_rttm() for a in anns)
        # one more tick with the outputs, through the recorder
        for sid, k in rec.sid_key.items():
            server.push(sid, np.zeros(8000, np.float32))
        rec.tick()
        recs.append((rec, last_windows(server, n)))
        launches.append(counts)
    assert launches[0] == launches[1], launches
    (a, wa), (b, wb) = recs
    assert np.array_equal(wa.view(np.uint32), wb.view(np.uint32))
    for k in range(n):
        assert a.rttm[k] == b.rttm[k]
        for sa, sb in ((a.seg, b.seg), (a.emb, b.emb), (a.maps, b.maps)):
            assert np.array_equal(np.stack(sa[k]), np.stack(sb[k]))


def test_refusals_leave_the_server_usable(oracle_nets, cuda_device):
    config = make_config(oracle_nets, cuda_device)
    server = MultiStreamDiarization(config, max_streams=2, max_windows_per_stream=2, source_sample_rates=(44100,))
    lib = _lib.lib()
    chunk, hop, res = source_geometry(44100, SR, 5.0, 0.5)
    a = source(6, 44100, 5)
    with pytest.raises(ValueError):                     # a rate that was not declared
        server.open(sample_rate=48000)
    sid = server.open(sample_rate=44100)
    server.push(sid, a[:chunk + hop])
    assert server.available(sid) == 2
    with pytest.raises(ValueError):                     # beyond the 44.1 kHz ring's capacity: refused, nothing written
        server.push(sid, np.zeros(chunk + 4 * hop, np.float32))
    assert server.available(sid) == 2
    rs = DeviceResample(48000, SR, cuda_device)
    rid = C.c_int()
    c48, h48, _ = source_geometry(48000, SR, 5.0, 0.5)
    assert lib.dg_multi_add_rate(server.handle, rs.handle, c48, h48, C.byref(rid)) == -1   # after an open
    with pytest.raises(ValueError):
        server.open(sample_rate=48000)
    # the windows are those of the audio
    got = server.step()[sid]
    x = Windows(cuda_device)(a, 44100, 0, 2)
    assert [g.to_rttm() for g in got] == dedicated(config, x, 0.0, res)[0]
