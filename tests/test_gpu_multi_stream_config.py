"""Per-stream latency and thresholds in the multi-stream servers (diart_b200.serve, dg_multi_open_config): every stream opened
with its own latency, tau_active, rho_update and delta_new gets exactly what a dedicated pipeline whose configuration is the
server's with those values gives on its windows fed one per call, whatever the other streams and their values are.

The diarization comparisons are those of test_gpu_multi_stream.py (scores, maps and RTTM bit for bit, embeddings within
EMB_TOL); the VAD comparisons are bit for bit."""
import math

import numpy as np
import pytest

from diart_b200 import _lib, blocks, synth
from diart_b200.serve import MultiStreamDiarization, MultiStreamVoiceActivityDetection, source_geometry
from oracle import nets
from test_gpu_multi_stream import EMB_TOL, Recorder, dedicated, make_config
from test_gpu_multi_stream_resampled import Windows, source
from test_gpu_multi_stream_vad import Recorder as VadRecorder
from test_gpu_multi_stream_vad import assert_same as assert_same_vad
from test_gpu_multi_stream_vad import dedicated as dedicated_vad
from test_gpu_multi_stream_vad import make_config as make_vad_config

pytestmark = pytest.mark.gpu

SR, S, HOP = 16000, 80000, 8000
# tau_active, rho_update, delta_new tuned per dataset (the reference README's table "To obtain the best results"): DIHARD III,
# AMI, VoxConverse, DIHARD II
README_ROWS = [(0.555, 0.422, 1.517), (0.507, 0.006, 1.057), (0.576, 0.915, 0.648), (0.619, 0.326, 0.997)]


def values(row):
    return dict(zip(("tau_active", "rho_update", "delta_new"), row))


def diarization_variant(config, **kw):
    """the server's configuration with a stream's own values, on the same model objects"""
    base = dict(latency=config.latency, tau_active=config.tau_active, rho_update=config.rho_update,
                delta_new=config.delta_new)
    return blocks.SpeakerDiarizationConfig(segmentation=config.segmentation, embedding=config.embedding,
                                           duration=config.duration, step=config.step, gamma=config.gamma,
                                           beta=config.beta, max_speakers=config.max_speakers,
                                           normalize_embedding_weights=config.normalize_embedding_weights,
                                           device=config.device, **{**base, **kw})


def vad_variant(config, **kw):
    base = dict(latency=config.latency, tau_active=config.tau_active)
    return blocks.VoiceActivityDetectionConfig(segmentation=config.segmentation, duration=config.duration, step=config.step,
                                               device=config.device, **{**base, **kw})


def run_ragged(server, rec, audio, plan, rng, count):
    """plan[k] = (windows, when, shift, open kwargs): `when` is the tick at which stream k opens, or ("after", j) for the tick
    after stream j closed.  Stream k is closed once it has `windows` results (count(rec, k)).  Ragged pushes, shorter than a
    hop or longer than a window, at each stream's own rate -> (windows per tick, [(stream, slot, slots freed before)])"""
    pos, sid_of, closed, reused = {}, {}, {}, []
    per_tick, tick = [], 0
    while len(closed) < len(plan):
        for k, (_, when, shift, kw) in enumerate(plan):
            if k in sid_of or k in closed:
                continue
            if when == tick or (isinstance(when, tuple) and when[1] in closed):
                sid_of[k] = server.open(shift, **kw)
                rec.sid_key[sid_of[k]] = k
                pos[k] = 0
                if isinstance(when, tuple):
                    reused.append((k, sid_of[k], set(closed.values())))
        for k, sid in list(sid_of.items()):
            a, chunk, hop = audio[k], int(server._chunk[sid]), int(server._hop[sid])
            room = chunk + 2 * server.max_windows_per_stream * hop - (server._pushed[sid] - server._emitted[sid] * hop)
            size = int(rng.integers(500, hop)) if rng.random() < 0.6 else int(rng.integers(chunk + 1, chunk + 3 * hop))
            size = min(size, room, len(a) - pos[k])
            if size > 0:
                server.push(sid, a[pos[k]:pos[k] + size])
                pos[k] += size
        per_tick.append(rec.tick())
        tick += 1
        for k, sid in list(sid_of.items()):
            if count(rec, k) >= plan[k][0]:
                server.close(sid)
                del sid_of[k]
                closed[k] = sid
        assert tick < 300
    return per_tick, reused


def assert_same_diarization(rec, k, want):
    rttm, seg, emb, maps = want
    n = len(rttm)
    assert rec.rttm[k][:n] == rttm, f"stream {k}: RTTM differs"
    assert np.array_equal(np.stack(rec.seg[k][:n]), seg), f"stream {k}: scores differ"
    assert np.abs(np.stack(rec.emb[k][:n]) - emb).max() <= EMB_TOL, f"stream {k}: embeddings differ"
    assert np.array_equal(np.stack(rec.maps[k][:n]), maps), f"stream {k}: speaker maps differ"


def test_diarization_streams_at_their_own_values(oracle_nets, cuda_device):
    config = make_config(oracle_nets, cuda_device, latency=1.0)
    rng = np.random.default_rng(23)
    same = dict(latency=2.0)
    # (windows, when, shift, open kwargs).  Stream 5 (latency 5) closes after 9 windows and stream 7 opens at 0.5 in a freed
    # slot; stream 6 (latency 0.5) closes after 11 and stream 8 opens at 5.  Streams 9 and 10 are the same audio at two
    # sets of thresholds.
    plan = [(30, 0, 0.0, dict(latency=5.0, **values(README_ROWS[0]))),
            (26, 0, 0.0, dict(latency=0.5, **values(README_ROWS[1]))),
            (22, 1, 3.25, dict(latency=1.0, **values(README_ROWS[2]))),
            (28, 2, 0.0, dict(latency=2.0, **values(README_ROWS[3]))),
            (24, 0, 1.5, dict()),
            (9, 0, 0.0, dict(latency=5.0, **values(README_ROWS[0]))),
            (11, 1, 0.0, dict(latency=0.5, **values(README_ROWS[1]))),
            (20, ("after", 5), 2.0, dict(latency=0.5, **values(README_ROWS[2]))),
            (16, ("after", 6), 0.0, dict(latency=5.0, **values(README_ROWS[3]))),
            (20, 0, 0.0, dict(same, tau_active=0.45, rho_update=0.1, delta_new=0.8)),
            (20, 3, 0.0, dict(same, tau_active=0.7, rho_update=0.5, delta_new=1.3))]
    audio = {k: synth.synth_audio(S + HOP * (n + 5), seed=1100 + k) for k, (n, _, _, _) in enumerate(plan)}
    audio[10] = audio[9]
    server = MultiStreamDiarization(config, max_streams=9, max_windows_per_stream=4, max_latency=5.0)
    assert server.nw == 10
    rec = Recorder(server)
    per_tick, reused = run_ragged(server, rec, audio, plan, rng, lambda r, k: len(r.rttm.get(k, [])))
    assert max(per_tick) > 6, per_tick
    assert sorted(k for k, _, _ in reused) == [7, 8] and all(sid in freed for _, sid, freed in reused), reused
    for k, (n, _, shift, kw) in enumerate(plan):
        assert_same_diarization(rec, k, dedicated(diarization_variant(config, **kw), audio[k], n, shift))
    assert rec.rttm[9][:20] != rec.rttm[10][:20], "the same audio at two sets of thresholds gave the same turns"


@pytest.mark.parametrize("powerset", [False, True], ids=["multilabel", "powerset"])
def test_vad_streams_at_their_own_values(oracle_nets, cuda_device, powerset):
    if powerset:
        config = make_vad_config(nets.make_powerset_segmentation().state_dict(), cuda_device, powerset=(3, 2), latency=1.0)
    else:
        config = make_vad_config(oracle_nets[0].state_dict(), cuda_device, latency=1.0)
    rate = 44100
    server = MultiStreamVoiceActivityDetection(config, max_streams=9, max_windows_per_stream=4, source_sample_rates=(rate,),
                                               max_latency=5.0)
    rng = np.random.default_rng(31 + powerset)
    plan = [(24, 0, 0.0, dict(latency=0.5, tau_active=0.45)),
            (26, 0, 2.5, dict()),
            (22, 1, 0.0, dict(latency=2.0, tau_active=0.7)),
            (28, 2, 0.0, dict(latency=5.0, tau_active=0.5)),
            (9, 0, 0.0, dict(latency=5.0, tau_active=0.55)),
            (11, 1, 0.0, dict(latency=0.5, tau_active=0.65)),
            (18, ("after", 4), 1.5, dict(latency=0.5, tau_active=0.4)),
            (14, ("after", 5), 0.0, dict(latency=5.0, tau_active=0.6)),
            (16, 0, 0.0, dict(latency=1.5, tau_active=0.35)),
            (16, 2, 0.0, dict(latency=1.5, tau_active=0.75)),
            (15, 0, 3.25, dict(sample_rate=rate, latency=1.5, tau_active=0.55))]
    audio = {k: synth.synth_audio(S + HOP * (n + 5), seed=1300 + k) for k, (n, _, _, _) in enumerate(plan)}
    audio[9] = audio[8]
    audio[10] = source(plan[10][0] + 5, rate, 1310)
    rec = VadRecorder(server)
    per_tick, reused = run_ragged(server, rec, audio, plan, rng, lambda r, k: len(r.anns.get(k, [])))
    assert max(per_tick) > 6, per_tick
    assert sorted(k for k, _, _ in reused) == [6, 7] and all(sid in freed for _, sid, freed in reused), reused
    for k, (n, _, shift, kw) in enumerate(plan):
        kw = dict(kw)
        if kw.pop("sample_rate", None):
            x = Windows(cuda_device)(audio[k], rate, 0, n)
            want = dedicated_vad(vad_variant(config, **kw), x, n, shift, source_geometry(rate, SR, 5.0, 0.5)[2])
        else:
            want = dedicated_vad(vad_variant(config, **kw), audio[k], n, shift)
        assert_same_vad(rec, k, want)
    assert rec.anns[8][:16] != rec.anns[9][:16], "the same audio at two thresholds gave the same turns"
    assert any(a[0] for k in rec.anns for a in rec.anns[k]), "no speech at all: the comparison says little"


def mixed(i):
    """stream i's open kwargs among many: the README rows and the defaults x latencies 0.5, 1, 2 and 5 s"""
    rows = README_ROWS + [None]
    row, latency = rows[(i // 4) % 5], (0.5, 1.0, 2.0, 5.0)[i % 4]
    return dict(latency=latency, **(values(row) if row else {}))


def run_streams(server, audios, kws, ticks):
    """every stream pushes its first window, then one hop per tick"""
    rec = Recorder(server)
    for k, kw in enumerate(kws):
        rec.sid_key[server.open(**kw)] = k
    for t in range(ticks):
        for sid, k in rec.sid_key.items():
            a = audios[k]
            server.push(sid, a[:S] if t == 0 else a[S + (t - 1) * HOP:S + t * HOP])
        rec.tick()
    return rec


def test_a_stream_alone_equals_it_among_300_of_mixed_values(oracle_nets, cuda_device):
    """300 windows per tick at 20 different configurations: two network sub-batches and more clustering states than one
    wave of CTAs.  Stream 149 (VoxConverse row at 1 s) sits at batch row 149 among 300, at row 0 alone; stream 275 (DIHARD
    II row at 5 s, a full history from tick 10 on) is in the second sub-batch and equals its dedicated pipeline"""
    config = make_config(oracle_nets, cuda_device, latency=2.0)
    ticks = 12
    base = [synth.synth_audio(S + HOP * (ticks - 1) + 40 * HOP, seed=1500 + i) for i in range(6)]
    audios = [np.ascontiguousarray(base[i % 6][(i // 6) % 40 * HOP:][:S + HOP * (ticks - 1)]) for i in range(300)]
    kws = [mixed(i) for i in range(300)]
    assert kws[149]["latency"] == 1.0 and kws[275]["latency"] == 5.0 and len({str(k) for k in kws}) == 20
    alone = run_streams(MultiStreamDiarization(config, 1, 1, max_latency=5.0), [audios[149]], [kws[149]], ticks)
    crowd = run_streams(MultiStreamDiarization(config, 300, 1, max_latency=5.0), audios, kws, ticks)
    assert len(crowd.rttm[149]) == ticks
    assert crowd.rttm[149] == alone.rttm[0]
    for store_c, store_a in ((crowd.seg, alone.seg), (crowd.maps, alone.maps)):
        assert np.array_equal(np.stack(store_c[149]), np.stack(store_a[0]))
    assert np.abs(np.stack(crowd.emb[149]) - np.stack(alone.emb[0])).max() <= EMB_TOL
    assert_same_diarization(crowd, 275, dedicated(diarization_variant(config, **kws[275]), audios[275], ticks))


class LegacyDiarization(MultiStreamDiarization):
    """a server whose streams open through dg_multi_open_rate, the entry point without per-stream values"""

    def open(self, shift=0.0, sample_rate=None):
        sid = int(np.flatnonzero(~self._open)[0])
        _lib.check(_lib.lib().dg_multi_open_rate(self._h, sid, -1))
        self._open[sid], self._pushed[sid], self._emitted[sid], self._shift[sid] = True, 0, 0, shift
        return sid


class LegacyVad(MultiStreamVoiceActivityDetection):
    open = LegacyDiarization.open


@pytest.mark.parametrize("kind", ["diarization", "vad"])
def test_defaults_run_the_launches_and_bits_of_today(oracle_nets, cuda_device, kind):
    """streams that pass nothing, and streams that pass the config's values, give the bits and issue the launches per tick
    of streams opened without per-stream values"""
    if kind == "diarization":
        config = make_config(oracle_nets, cuda_device, latency=1.5, tau_active=0.55, rho_update=0.25, delta_new=0.9)
        server_cls, legacy_cls, rec_cls = MultiStreamDiarization, LegacyDiarization, Recorder
        explicit = dict(latency=1.5, tau_active=0.55, rho_update=0.25, delta_new=0.9)
    else:
        config = make_vad_config(oracle_nets[0].state_dict(), cuda_device, latency=1.5, tau_active=0.55)
        server_cls, legacy_cls, rec_cls = MultiStreamVoiceActivityDetection, LegacyVad, VadRecorder
        explicit = dict(latency=1.5, tau_active=0.55)
    lib = _lib.lib()
    n_streams, ticks = 5, 8
    audios = [synth.synth_audio(S + HOP * (3 * ticks), seed=1700 + i) for i in range(n_streams)]
    results, launches = [], []
    for make, kw in ((lambda: legacy_cls(config, n_streams), {}), (lambda: server_cls(config, n_streams), {}),
                     (lambda: server_cls(config, n_streams, max_latency=1.5), explicit)):
        server = make()
        rec = rec_cls(server)
        for k in range(n_streams):
            rec.sid_key[server.open(0.5 * k, **kw)] = k
        per_tick = []
        for t in range(ticks):
            for sid, k in rec.sid_key.items():
                a = audios[k]
                # 1 to 3 windows per stream and tick: 1 + (u + k) % 3 in tick u
                lo = 0 if t == 0 else S + HOP * (sum(1 + (u + k) % 3 for u in range(t)) - 1)
                hi = S + HOP * (sum(1 + (u + k) % 3 for u in range(t + 1)) - 1)
                server.push(sid, a[lo:hi])
            before = lib.dg_launch_count()
            rec.tick()
            per_tick.append(lib.dg_launch_count() - before)
        results.append(rec)
        launches.append(per_tick)
    assert launches[0] == launches[1] == launches[2], launches
    stores = ("rttm", "seg", "emb", "maps") if kind == "diarization" else ("anns", "seg")
    for other in results[1:]:
        for name in stores:
            want, got = getattr(results[0], name), getattr(other, name)
            assert sorted(want) == sorted(got)
            for k in want:
                if name in ("rttm", "anns"):
                    assert got[k] == want[k], f"{name} of stream {k}"
                else:
                    assert np.array_equal(np.stack(got[k]), np.stack(want[k])), f"{name} of stream {k}"


def test_refusals_launch_nothing_and_leave_the_slot_closed(oracle_nets, cuda_device):
    config = make_config(oracle_nets, cuda_device, latency=2.0)
    server = MultiStreamDiarization(config, max_streams=2, max_windows_per_stream=2, max_latency=5.0)
    vad = MultiStreamVoiceActivityDetection(make_vad_config(oracle_nets[0].state_dict(), cuda_device, latency=2.0), 2,
                                            max_latency=3.0)
    lib = _lib.lib()
    before = lib.dg_launch_count()
    for kw in (dict(latency=0.25), dict(latency=5.5), dict(tau_active=math.nan), dict(rho_update=math.inf),
               dict(delta_new=-math.inf)):
        with pytest.raises(ValueError):
            server.open(**kw)
    for kw in (dict(latency=3.5), dict(tau_active=math.inf)):
        with pytest.raises(ValueError):
            vad.open(**kw)
    for kw in (dict(rho_update=0.3), dict(delta_new=1.0)):
        with pytest.raises(TypeError):
            vad.open(**kw)
    good = np.array([0.5, 0.3, 1.0])
    for nw, params in ((server.nw + 1, good), (0, good), (4, np.array([0.5, math.nan, 1.0]))):
        assert lib.dg_multi_open_config(server.handle, 0, -1, nw, params.ctypes.data) == -1
        assert b"dg_multi_open_config" in lib.dg_last_error()
    assert lib.dg_multi_open_config(vad.handle, 0, -1, vad.nw + 1, good.ctypes.data) == -1
    assert lib.dg_launch_count() == before
    for s in (server, vad):
        assert not s._open.any()
        for slot in (0, 1):
            assert lib.dg_multi_available(s.handle, slot) == -1              # still closed
    # a VAD handle reads only params[0]
    assert lib.dg_multi_open_config(vad.handle, 0, -1, 2, np.array([0.5, math.nan, math.nan]).ctypes.data) == 0
    assert lib.dg_multi_close(vad.handle, 0) == 0
    # the servers are still usable, at the stream's own values
    a = synth.synth_audio(S + 2 * HOP, seed=9)
    sid = server.open(latency=0.5, **values(README_ROWS[1]))
    assert sid == 0
    server.push(sid, a)
    got = [g.to_rttm() for g in server.step()[sid]]
    assert got == dedicated(diarization_variant(config, latency=0.5, **values(README_ROWS[1])), a, 2)[0]
