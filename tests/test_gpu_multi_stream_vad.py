"""Many live VAD streams on one device (diart_b200.serve.MultiStreamVoiceActivityDetection, dg_multi_create_vad): every stream
gets exactly what a dedicated VoiceActivityDetection gives on its windows fed one per call (the reference's live mode), whatever
the other streams do in the same ticks.

Everything is compared bit for bit: the segmentation scores are batch invariant, and the speech curve is the post-path's
arithmetic with one speaker, so there is no tolerance anywhere in this file."""
import ctypes as C
import json

import numpy as np
import pytest
import torch

from diart_b200 import _lib, blocks, models, synth
from diart_b200.core import SlidingWindow, SlidingWindowFeature
from diart_b200.serve import MultiStreamDiarization, MultiStreamVoiceActivityDetection, plan_rows, source_geometry
from oracle import nets
from test_gpu_multi_stream_resampled import Windows, last_windows, source

pytestmark = pytest.mark.gpu

SR, S, HOP = 16000, 80000, 8000


def make_config(state, device, powerset=None, **kw):
    return blocks.VoiceActivityDetectionConfig(
        segmentation=models.SegmentationModel(models.B200SegmentationLoader(state, powerset=powerset)), device=device, **kw)


def window(x, i, res=1 / SR):
    """window i of a stream (x: its samples), or x[i] when x is already a stack of windows"""
    data = x[i] if x.ndim == 2 else x[i * HOP:i * HOP + S]
    return SlidingWindowFeature(data[:, None], SlidingWindow(start=i * 0.5, duration=res, step=res))


def dedicated(config, x, n, shift=0.0, res=1 / SR):
    """the reference's live mode: a VoiceActivityDetection per stream, one window per call -> (per window (RTTM, uri,
    modality)), and each window's scores from SpeakerSegmentation.forward_device on that window alone"""
    pipe = blocks.VoiceActivityDetection(config)
    pipe.set_timestamp_shift(shift)
    seg = blocks.SpeakerSegmentation(config.segmentation, config.device)
    anns, scores = [], []
    for i in range(n):
        a = pipe([window(x, i, res)])[0][0]
        anns.append((a.to_rttm(), a.uri, a.modality))
        w = x[i:i + 1] if x.ndim == 2 else synth.windows(x, 1, first=i)
        scores.append(seg.forward_device(torch.from_numpy(np.ascontiguousarray(w))).cpu().numpy()[0])
    return anns, np.stack(scores)


class Recorder:
    """runs ticks of a server and keeps, per stream key, its annotations and its rows of the tick's scores"""

    def __init__(self, server):
        self.server, self.anns, self.seg, self.sid_key = server, {}, {}, {}

    def tick(self):
        res, outs = self.server._step(outputs=True)
        seg = outs[0].cpu().numpy() if outs else None
        r = 0
        for sid in sorted(res):
            key, n = self.sid_key[sid], len(res[sid])
            self.anns.setdefault(key, []).extend((a.to_rttm(), a.uri, a.modality) for a in res[sid])
            self.seg.setdefault(key, []).extend(seg[r:r + n])
            r += n
        return r


def assert_same(rec, k, want):
    anns, seg = want
    n = len(anns)
    assert rec.anns[k][:n] == anns, f"stream {k}: annotations differ"
    assert np.array_equal(np.stack(rec.seg[k][:n]).view(np.uint32), seg.view(np.uint32)), f"stream {k}: scores differ"


def run_ragged(server, audio, plan, rng, close_after=None):
    """plan: per stream (windows, tick at which it opens or None, timestamp shift); stream close_after[0] is closed after
    close_after[1] windows, and the stream whose tick is None then opens in its slot.  Ragged pushes (shorter than a hop,
    longer than a window) -> the recorder and the windows per tick"""
    rec = Recorder(server)
    pos, sid_of, done, closed_sid = {}, {}, set(), None
    per_tick, tick = [], 0
    while len(done) < len(plan):
        for k, (n, t_open, shift) in enumerate(plan):
            if k not in sid_of and k not in done and (t_open == tick or (t_open is None and closed_sid is not None)):
                sid_of[k] = server.open(shift)
                rec.sid_key[sid_of[k]] = k
                pos[k] = 0
                if t_open is None:
                    assert sid_of[k] == closed_sid, "the new stream takes the closed stream's slot"
        for k, sid in list(sid_of.items()):
            a = audio[k]
            room = server.window_samples + 2 * server.max_windows_per_stream * HOP - \
                (server._pushed[sid] - server._emitted[sid] * HOP)
            size = int(rng.integers(500, HOP)) if rng.random() < 0.6 else int(rng.integers(S + 1, S + 30000))
            size = min(size, room, len(a) - pos[k])
            if size > 0:
                server.push(sid, a[pos[k]:pos[k] + size][None, :] if rng.random() < 0.5 else a[pos[k]:pos[k] + size])
                pos[k] += size
        per_tick.append(rec.tick())
        tick += 1
        for k, sid in list(sid_of.items()):
            got = len(rec.anns.get(k, []))
            if (close_after and k == close_after[0] and got >= close_after[1]) or got == plan[k][0]:
                server.close(sid)
                del sid_of[k]
                done.add(k)
                if close_after and k == close_after[0]:
                    closed_sid = sid
        assert tick < 300
    return rec, per_tick


@pytest.mark.parametrize("kw", [dict(latency=0.5), dict(latency=2.0), dict(latency=5.0), dict(latency=2.0, tau_active=0.45)],
                         ids=["latency0.5", "latency2", "latency5", "tau0.45"])
def test_streams_equal_dedicated_pipelines(oracle_nets, cuda_device, kw):
    config = make_config(oracle_nets[0].state_dict(), cuda_device, **kw)
    rng = np.random.default_rng(11)
    # (seed, windows, tick at which the stream opens, timestamp shift); stream 1 is closed after 9 windows and stream 6
    # then opens in its slot
    seeds = [101, 102, 103, 104, 105, 106, 107]
    plan = [(40, 0, 0.0), (70, 0, 0.0), (33, 2, 3.25), (45, 5, 0.0), (20, 1, 0.0), (52, 3, 0.0), (24, None, 1.5)]
    audio = {k: synth.synth_audio(S + HOP * (n - 1), seed=seeds[k]) for k, (n, _, _) in enumerate(plan)}
    server = MultiStreamVoiceActivityDetection(config, max_streams=6, max_windows_per_stream=4)
    rec, per_tick = run_ragged(server, audio, plan, rng, close_after=(1, 9))
    assert 0 in per_tick and max(per_tick) > 6, per_tick
    for k, (n, _, shift) in enumerate(plan):
        assert_same(rec, k, dedicated(config, audio[k], 9 if k == 1 else n, shift))
    assert any(a[0] for k in rec.anns for a in rec.anns[k]), "no speech at all: the comparison says little"


def test_powerset_segmentation(cuda_device):
    net = nets.make_powerset_segmentation()
    config = make_config(net.state_dict(), cuda_device, powerset=(3, 2), latency=2.0)
    assert config.segmentation.to(cuda_device).model.dims(S) == (293, 3)
    rng = np.random.default_rng(29)
    plan = [(18, 0, 0.0), (14, 1, 2.5), (21, 0, 0.0)]
    audio = {k: synth.synth_audio(S + HOP * (n - 1), seed=900 + k) for k, (n, _, _) in enumerate(plan)}
    server = MultiStreamVoiceActivityDetection(config, max_streams=3, max_windows_per_stream=4)
    rec, _ = run_ragged(server, audio, plan, rng)
    for k, (n, _, shift) in enumerate(plan):
        assert_same(rec, k, dedicated(config, audio[k], n, shift))


def test_streams_at_other_rates(oracle_nets, cuda_device):
    """16, 44.1 and 48 kHz streams in the same ticks: every resampled row of a tick has the bits of DeviceResample on the
    stacked source windows, and every stream equals a dedicated pipeline fed those windows in the resampled time base"""
    config = make_config(oracle_nets[0].state_dict(), cuda_device, latency=1.5)
    rates = (44100, 48000)
    server = MultiStreamVoiceActivityDetection(config, max_streams=5, max_windows_per_stream=4, source_sample_rates=rates)
    ref = Windows(cuda_device)
    rng = np.random.default_rng(5)
    plan = [(44100, 14, 0.0), (SR, 12, 1.5), (48000, 13, 3.25), (44100, 11, 0.0), (48000, 15, 2.0)]
    audio = {k: source(n, r, 450 + k) for k, (r, n, _) in enumerate(plan)}
    rec = Recorder(server)
    sid = {}
    for k, (r, _, shift) in enumerate(plan):
        sid[k] = server.open(shift=shift, sample_rate=r)
        rec.sid_key[sid[k]] = k
    pos = {k: 0 for k in sid}
    checked = 0
    for _ in range(100):
        for k, (r, _, _) in enumerate(plan):
            chunk, hop, _ = source_geometry(r, SR, 5.0, 0.5)
            room = chunk + 8 * hop - (server._pushed[sid[k]] - server._emitted[sid[k]] * hop)
            size = int(rng.integers(300, hop)) if rng.random() < 0.6 else int(rng.integers(chunk + 1, chunk + 2 * hop))
            size = min(size, room, len(audio[k]) - pos[k])
            if size > 0:
                server.push(sid[k], audio[k][pos[k]:pos[k] + size])
                pos[k] += size
        before = server._emitted.copy()
        B = rec.tick()
        if B:
            got, r0 = last_windows(server, B), 0
            for k in sorted(sid, key=lambda k: sid[k]):
                n = int(server._emitted[sid[k]] - before[sid[k]])
                if not n:
                    continue
                want = ref(audio[k], plan[k][0], int(before[sid[k]]), n)
                assert np.array_equal(got[r0:r0 + n].view(np.uint32), want.view(np.uint32)), f"stream {k}"
                r0 += n
                checked += n
        if all(len(rec.anns.get(k, [])) == n for k, (_, n, _) in enumerate(plan)):
            break
    assert checked == sum(n for _, n, _ in plan)
    for k, (r, n, shift) in enumerate(plan):
        x = ref(audio[k], r, 0, n)
        assert_same(rec, k, dedicated(config, x, n, shift, source_geometry(r, SR, 5.0, 0.5)[2]))


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
    """300 windows per tick: two segmentation sub-batches, one on each scratch lane.  Stream 137 sits at batch row 137 among
    300, at row 0 alone; stream 280 is in the second sub-batch"""
    config = make_config(oracle_nets[0].state_dict(), cuda_device, latency=2.0)
    ticks = 5
    base = [synth.synth_audio(S + HOP * (ticks - 1) + 40 * HOP, seed=300 + i) for i in range(6)]
    audios = [np.ascontiguousarray(base[i % 6][(i // 6) % 40 * HOP:][:S + HOP * (ticks - 1)]) for i in range(300)]
    alone = run_streams(MultiStreamVoiceActivityDetection(config, max_streams=1, max_windows_per_stream=1), [audios[137]],
                        ticks)
    crowd = run_streams(MultiStreamVoiceActivityDetection(config, max_streams=300, max_windows_per_stream=1), audios, ticks)
    assert len(crowd.anns[137]) == ticks and crowd.anns[137] == alone.anns[0]
    assert np.array_equal(np.stack(crowd.seg[137]), np.stack(alone.seg[0]))
    assert_same(crowd, 280, dedicated(config, audios[280], ticks))     # a row of the second sub-batch


class Capture(MultiStreamVoiceActivityDetection):
    """keeps the raw header and turns of every tick"""

    def _annotations(self, header, turns, n_turns, out_start, out_res, shifts):
        self.raw = (header.copy(), turns[:n_turns].copy())
        return super()._annotations(header, turns, n_turns, out_start, out_res, shifts)


@pytest.mark.parametrize("latency", [1.0, 5.0])
def test_the_kernel_equals_the_post_path_on_max_curves(oracle_nets, cuda_device, latency):
    """vad_slots' headers (count, frames) and packed turns equal dg_post_step with K = M = 1 on amax of the same scores, with
    the same plan rows and one post-path handle (history) per stream.  At latency 5 the history holds 9 entries, the most."""
    config = make_config(oracle_nets[0].state_dict(), cuda_device, latency=latency)
    server = Capture(config, max_streams=4, max_windows_per_stream=3)
    lib = _lib.lib()
    rng = np.random.default_rng(int(latency * 10))
    n_win = 16
    audio = [synth.synth_audio(S + HOP * (n_win - 1), seed=700 + k) for k in range(4)]
    sids = [server.open() for _ in range(4)]
    post = [blocks.post.DevicePostPath(0.5, latency, config.tau_active, server.F, 1, 1, cuda_device) for _ in sids]
    pos, done = [0] * 4, 0
    full_history = False
    for _ in range(100):
        for k, sid in enumerate(sids):
            size = min(int(rng.integers(2000, 3 * HOP)), len(audio[k]) - pos[k],
                       S + 6 * HOP - int(server._pushed[sid] - server._emitted[sid] * HOP))
            if size > 0:
                server.push(sid, audio[k][pos[k]:pos[k] + size])
                pos[k] += size
        before = server._emitted.copy()
        res, outs = server._step(outputs=True)
        if not res:
            continue
        (seg,) = outs
        header, turns = server.raw
        vad = seg.amax(dim=-1, keepdim=True).contiguous()
        r0 = 0
        for k, sid in enumerate(sids):
            n = int(server._emitted[sid] - before[sid])
            if not n:
                continue
            idx = before[sid] + np.arange(n)
            plan, _, _ = plan_rows(idx, 0.5, S, SR, server.F, server.nw, latency)
            plan = np.ascontiguousarray(plan)
            full_history |= server.nw == 10 and idx[0] >= 9          # its first row reads 9 history entries
            h, t = np.empty((n, 4), np.int32), np.empty(n * ((server.F + 2) // 2), np.uint32)
            nt = C.c_int()
            maps = torch.zeros((n, 1), dtype=torch.int32, device=cuda_device)
            with torch.cuda.device(cuda_device):
                _lib.check(lib.dg_post_step(post[k].handle, vad[r0:r0 + n].data_ptr(), maps.data_ptr(), n, plan.ctypes.data,
                                            h.ctypes.data, t.ctypes.data, len(t), C.byref(nt), _lib.stream_ptr(cuda_device)))
            torch.cuda.synchronize(cuda_device)
            for i in range(n):
                got_h = header[r0 + i]
                assert (got_h[1], got_h[2]) == (h[i, 1], h[i, 2]), f"stream {k}, window {idx[i]}"
                assert np.array_equal(turns[got_h[0]:got_h[0] + got_h[1]], t[h[i, 0]:h[i, 0] + h[i, 1]]), \
                    f"stream {k}, window {idx[i]}"
            r0 += n
            done += n
        if done == 4 * n_win:
            break
    assert done == 4 * n_win
    assert full_history or latency != 5.0


def test_shared_model_objects_interleaved(oracle_nets, cuda_device):
    """a VAD server, a diarization server and a VoiceActivityDetection on the same segmentation model object, calls
    interleaved: each gives its solo results"""
    seg_o, emb_o = oracle_nets
    seg_model = models.SegmentationModel(models.B200SegmentationLoader(seg_o.state_dict()))
    vad_cfg = blocks.VoiceActivityDetectionConfig(segmentation=seg_model, latency=1.5, device=cuda_device)
    dia_cfg = blocks.SpeakerDiarizationConfig(
        segmentation=seg_model, embedding=models.EmbeddingModel(models.B200EmbeddingLoader(emb_o.state_dict())),
        latency=1.5, device=cuda_device)
    n = 12
    a_vad, a_dia, a_pipe = (synth.synth_audio(S + HOP * (n - 1), seed=s) for s in (81, 82, 83))

    def block(a, i):
        return a[:S] if i == 0 else a[S + (i - 1) * HOP:S + i * HOP]

    solo_vad = run_streams(MultiStreamVoiceActivityDetection(vad_cfg, 2), [a_vad], n).anns[0]
    dia = MultiStreamDiarization(dia_cfg, 2)
    sid = dia.open()
    solo_dia = []
    for i in range(n):
        dia.push(sid, block(a_dia, i))
        solo_dia += [a.to_rttm() for a in dia.step()[sid]]
    solo_pipe = dedicated(vad_cfg, a_pipe, n)[0]
    vad_srv, dia_srv, pipe = MultiStreamVoiceActivityDetection(vad_cfg, 2), MultiStreamDiarization(dia_cfg, 2), \
        blocks.VoiceActivityDetection(vad_cfg)
    sv, sd = vad_srv.open(), dia_srv.open()
    got_vad, got_dia, got_pipe = [], [], []
    for i in range(n):
        vad_srv.push(sv, block(a_vad, i))
        dia_srv.push(sd, block(a_dia, i))
        got_vad += [(a.to_rttm(), a.uri, a.modality) for a in vad_srv.step()[sv]]
        got_pipe.append(pipe([window(a_pipe, i)])[0][0])
        got_dia += [a.to_rttm() for a in dia_srv.step()[sd]]
    assert got_vad == solo_vad and got_dia == solo_dia
    assert [(a.to_rttm(), a.uri, a.modality) for a in got_pipe] == solo_pipe


def profile_report():
    buf = C.create_string_buffer(1 << 16)
    n = _lib.lib().dg_profile_report(buf, len(buf))
    assert n >= 0
    return json.loads(buf.value.decode())


def test_no_embedding_or_clustering_work_and_refusals(oracle_nets, cuda_device):
    config = make_config(oracle_nets[0].state_dict(), cuda_device, latency=1.0)
    server = MultiStreamVoiceActivityDetection(config, max_streams=2, max_windows_per_stream=2, source_sample_rates=(44100,))
    lib = _lib.lib()
    a = synth.synth_audio(S + 4 * HOP, seed=5)
    sid = server.open()
    server.push(sid, a[:S + HOP])
    assert server.available(sid) == 2
    # what a VAD tick runs
    profile_report()
    lib.dg_profile_enable(1)
    try:
        got = server.step()[sid]
        tags = profile_report()
    finally:
        lib.dg_profile_enable(0)
    assert {"ring_scatter", "ring_gather", "vad_slots", "vad_slots_history"} <= set(tags), tags
    forbidden = ("osp", "pool_weights", "pool_finalize", "l2norm", "tdnn", "cluster_sweep", "post_slots", "post_slots_history")
    assert not [t for t in tags if t.startswith(forbidden)], tags
    assert [(g.to_rttm(), g.uri, g.modality) for g in got] == dedicated(config, a, 2)[0]
    # refusals
    server.push(sid, a[S + HOP:S + 2 * HOP])
    assert server.available(sid) == 1
    with pytest.raises(ValueError):                     # more than the ring holds: refused, nothing staged
        server.push(sid, np.zeros(S + 4 * HOP, np.float32))
    assert server.available(sid) == 1
    with pytest.raises(ValueError):                     # unknown slot
        server.push(7, a[:10])
    with pytest.raises(ValueError):                     # a rate that was not declared
        server.open(sample_rate=48000)
    other = server.open()
    server.close(other)
    with pytest.raises(ValueError):                     # closed slot
        server.push(other, a[:10])
    with pytest.raises(ValueError):
        server.available(other)
    counts, header, turns, nt = np.empty(2, np.int32), np.empty((4, 4), np.int32), np.empty(4096, np.uint32), C.c_int()
    plan = np.ascontiguousarray(plan_rows(np.array([2]), 0.5, S, SR, server.F, server.nw, 1.0)[0])
    junk = torch.empty(64, device=cuda_device)
    before = lib.dg_launch_count()
    for emb, maps in ((junk.data_ptr(), None), (None, junk.data_ptr())):   # a VAD handle has no embeddings or maps
        assert lib.dg_multi_step(server.handle, plan.ctypes.data, 1, counts.ctypes.data, header.ctypes.data,
                                 turns.ctypes.data, len(turns), C.byref(nt), None, emb, maps) == -1
        assert b"VAD" in lib.dg_last_error()
    wide = np.zeros((2, 4 + server.nw), np.int32)                          # a plan for another number of windows
    assert lib.dg_multi_step(server.handle, wide.ctypes.data, 2, counts.ctypes.data, header.ctypes.data, turns.ctypes.data,
                             len(turns), C.byref(nt), None, None, None) == -1
    assert lib.dg_launch_count() == before
    # the server is still usable, and its windows are those of the audio
    got = server.step()[sid]
    assert [(g.to_rttm(), g.uri, g.modality) for g in got] == dedicated(config, a, 3)[0][2:]
    # a tick without windows launches nothing
    before = lib.dg_launch_count()
    assert server.step() == {}
    assert lib.dg_launch_count() == before
    # a segmentation model that is not the native one
    foreign = blocks.VoiceActivityDetectionConfig(segmentation=models.SegmentationModel(lambda: torch.nn.Identity()),
                                                  device=cuda_device)
    with pytest.raises(_lib.DiartB200Error):
        MultiStreamVoiceActivityDetection(foreign, 2)
