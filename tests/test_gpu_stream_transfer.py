"""Moving live streams between servers (export / restore): a moved stream continues exactly as the same stream on one server
that never exported it ("uninterrupted": the same pushes and the same tick schedule).

RTTM, scores and speaker maps are compared bit for bit, embeddings within EMB_TOL (a window's embedding depends on its row
in the batch, see tests/test_gpu_multi_stream.py); a stream alone on both servers gives bit-identical embeddings and
centroids."""

import numpy as np
import pytest
import torch

from diart_b200 import _lib, blocks, models, synth
from diart_b200.serve import MultiStreamDiarization, MultiStreamVoiceActivityDetection
from diart_b200.speakers import KnownSpeakers, SpeakerGallery
from diart_b200.transfer import StreamState
from test_gpu_multi_stream import EMB_TOL, HOP, S, make_config

pytestmark = pytest.mark.gpu


def vad_config(oracle_nets, device, **kw):
    return blocks.VoiceActivityDetectionConfig(segmentation=make_config(oracle_nets, device).segmentation, device=device, **kw)


def schedule(n_streams, ticks, seed, rate=16000):
    """ragged pushes per tick and stream: shorter than a hop or longer than a window, at most 4 windows' worth ahead"""
    rng = np.random.default_rng(seed)
    hop, win = HOP * rate // 16000, S * rate // 16000
    return [[int(rng.integers(200, hop)) if rng.random() < 0.6 else int(rng.integers(win + 1, win + 3 * hop))
             for _ in range(n_streams)] for _ in range(ticks)]


class Run:
    """drives streams on a server; a stream may move (export, then restore in `target`, another slot or server) at a
    tick, before that tick's step (its last pushes staged) or after it.  Records per stream key its RTTM, scores,
    embeddings, maps, window rows and (alone) centroids per tick."""

    def __init__(self, server, audios, sched, open_kw=None, keep=None, replay=None):
        self.servers, self.audios, self.sched, self.keep = [server], audios, sched, keep
        self.replay = None if replay is None else replay.pushed
        self.pushed = {}
        self.where = {}   # key -> (server index, sid)
        for k in range(len(audios)):
            self.where[k] = (0, server.open(**(open_kw[k] if open_kw else {})))
        self.pos = {k: 0 for k in self.where}
        self.rttm, self.seg, self.emb, self.maps, self.wav, self.cent = ({} for _ in range(6))

    def push(self, t):
        """the scheduled blocks, as far as the ring has room; a Run given another's `pushed` pushes exactly what that one
        did (a target with more room must not change the audio)"""
        for k, (i, sid) in self.where.items():
            srv = self.servers[i]
            room = srv._chunk[sid] + 2 * srv.max_windows_per_stream * srv._hop[sid] - (
                srv._pushed[sid] - srv._emitted[sid] * srv._hop[sid])
            n = min(self.sched[t][k], room, len(self.audios[k]) - self.pos[k])
            if self.replay is not None:
                n = self.replay.get((t, k), 0)
            self.pushed[(t, k)] = n
            if n > 0:
                srv.push(sid, self.audios[k][self.pos[k]:self.pos[k] + n])
                self.pos[k] += n

    def step(self):
        for i, srv in enumerate(self.servers):
            res, outs = srv._step(outputs=True)
            if not res:
                continue
            B = sum(len(v) for v in res.values())
            wav = torch.empty((B, srv.window_samples), device=srv.device)
            _lib.check(_lib.lib().dg_multi_last_windows(srv.handle, wav.data_ptr(), B))
            arrs = [t.cpu().numpy() for t in outs] + [wav.cpu().numpy()]
            r = 0
            for sid in sorted(res):
                n = len(res[sid])
                key = next(k for k, v in self.where.items() if v == (i, sid))
                if self.keep is not None and key not in self.keep:
                    r += n
                    continue
                self.rttm.setdefault(key, []).extend(a.to_rttm() for a in res[sid])
                stores = (self.seg, self.emb, self.maps, self.wav) if len(arrs) == 4 else (self.seg, self.wav)
                for store, arr in zip(stores, arrs):
                    store.setdefault(key, []).extend(arr[r:r + n])
                r += n
                if isinstance(srv, MultiStreamDiarization):
                    self.cent.setdefault(key, []).append(srv.speakers(sid).centroids.copy())

    def move(self, key, target=None, restore_kw=None, via_file=None):
        i, sid = self.where[key]
        src = self.servers[i]
        state = src.export([sid])[0]
        if via_file is not None:
            state.save(via_file)
            state = StreamState.load(via_file)
        if target is None:   # another slot of the same server: placeholders take the free slots up to the freed one
            holds = [src.open()]
            while holds[-1] != sid:
                holds.append(src.open())
            self.where[key] = (i, src.restore([state], **(restore_kw or {}))[0])
            assert self.where[key][1] != sid
            for h in holds:
                src.close(h)
        else:
            if target not in self.servers:
                self.servers.append(target)
            self.where[key] = (self.servers.index(target), target.restore([state], **(restore_kw or {}))[0])

    def go(self, moves=()):
        """moves: {(tick, "before" | "after"): [(key, target or None, restore kwargs)]}"""
        moves = dict(moves)
        for t in range(len(self.sched)):
            self.push(t)
            for key, target, kw in moves.get((t, "before"), []):
                self.move(key, target, kw)
            self.step()
            for key, target, kw in moves.get((t, "after"), []):
                self.move(key, target, kw)
        return self.drain()

    def drain(self, after_step=lambda: None):
        """ticks until the audio pushed is consumed"""
        for _ in range(60):
            if not any(self.servers[i].available(sid) for i, sid in self.where.values()):
                break
            self.step()
            after_step()
        return self


def same(a, b, keys, emb_exact=False):
    for k in keys:
        assert a.rttm[k] == b.rttm[k], f"stream {k}: RTTM differs"
        assert np.array_equal(np.stack(a.seg[k]), np.stack(b.seg[k])), f"stream {k}: scores differ"
        assert np.array_equal(np.stack(a.wav[k]), np.stack(b.wav[k])), f"stream {k}: windows differ"
        if k in a.maps:
            assert np.array_equal(np.stack(a.maps[k]), np.stack(b.maps[k])), f"stream {k}: maps differ"
            d = np.abs(np.stack(a.emb[k]) - np.stack(b.emb[k])).max()
            assert (d == 0) if emb_exact else d <= EMB_TOL, f"stream {k}: embeddings differ by {d}"
        if emb_exact and k in a.cent:
            for x, y in zip(a.cent[k], b.cent[k]):
                assert np.array_equal(x, y), f"stream {k}: centroids differ"


TICKS = 14


@pytest.mark.parametrize("kw", [dict(latency=0.5), dict(latency=2.0), dict(latency=2.0, max_speakers=4)],
                         ids=["latency0.5", "latency2", "speakers4"])
def test_diarization_continues_exactly(oracle_nets, cuda_device, kw):
    config = make_config(oracle_nets, cuda_device, **kw)
    audios = [synth.synth_audio(S + HOP * 60, seed=500 + k) for k in range(6)]
    sched = schedule(6, TICKS, seed=9)
    sched[0][3] = 3000   # stream 3 moves before its first window is complete
    mk = lambda: MultiStreamDiarization(config, max_streams=8, max_windows_per_stream=4)  # noqa: E731
    want = Run(mk(), audios, sched).go()
    other = MultiStreamDiarization(config, max_streams=11, max_windows_per_stream=6, max_latency=3.0,
                                   source_sample_rates=(44100,))
    got = Run(mk(), audios, sched, replay=want).go({(0, "after"): [(3, None, None)], (4, "after"): [(1, None, None)],
                                       (6, "before"): [(2, other, None)], (8, "after"): [(1, other, None)],
                                       (10, "before"): [(2, None, None)]})
    assert all(len(want.rttm[k]) > 8 for k in range(6))
    same(want, got, range(6))


def test_a_stream_alone_is_bit_identical(oracle_nets, cuda_device):
    config = make_config(oracle_nets, cuda_device, latency=2.0)
    audios = [synth.synth_audio(S + HOP * 40, seed=77)]
    sched = schedule(1, TICKS, seed=2)
    want = Run(MultiStreamDiarization(config, 2), audios, sched).go()
    other = MultiStreamDiarization(config, 3, max_latency=3.0)
    got = Run(MultiStreamDiarization(config, 2), audios, sched, replay=want).go({(3, "before"): [(0, other, None)]})
    same(want, got, [0], emb_exact=True)


def test_resampled_streams(oracle_nets, cuda_device):
    config = make_config(oracle_nets, cuda_device, latency=1.5)
    rates = (44100, 48000)
    audios = [synth.synth_audio((S + HOP * 40) * r // 16000, seed=40 + k, sample_rate=r) for k, r in enumerate(rates)]
    sched = [[max(1, b * r // 16000) for b, r in zip(row, rates)] for row in schedule(2, TICKS, seed=5)]
    kw = [dict(sample_rate=r) for r in rates]
    want = Run(MultiStreamDiarization(config, 3, source_sample_rates=rates), audios, sched, kw).go()
    other = MultiStreamDiarization(config, 4, max_windows_per_stream=7, source_sample_rates=rates + (22050,))
    got = Run(MultiStreamDiarization(config, 3, source_sample_rates=rates), audios, sched, kw, replay=want).go(
        {(4, "before"): [(0, other, None)], (5, "after"): [(1, other, None)]})
    assert all(len(want.rttm[k]) > 5 for k in range(2))
    same(want, got, range(2))


def test_known_speakers_and_galleries(oracle_nets, cuda_device):
    """seeded streams named from their own gallery and from the server default keep their names and claims"""
    config = make_config(oracle_nets, cuda_device, latency=1.0)
    audios = [synth.synth_audio(S + HOP * 40, seed=90 + k) for k in range(3)]
    sched = schedule(3, TICKS, seed=12)
    probe = MultiStreamDiarization(config, 3)
    learned = Run(probe, audios, [[n for n in row] for row in sched[:6]])
    learned.go()
    cents = [probe.speakers(sid).centroids for _, sid in learned.where.values()]
    rows = np.concatenate([c for c in cents if len(c)])
    assert len(rows) >= 2
    names = [f"person{e}" for e in range(len(rows))]
    gal = SpeakerGallery(KnownSpeakers(names, rows + 1e-3), threshold=1.0, device=cuda_device)
    own = SpeakerGallery(KnownSpeakers(names[::-1], rows[::-1] * 1.01), threshold=0.8, device=cuda_device)
    seed = KnownSpeakers(["person0"], rows[:1])
    open_kw = [dict(gallery=own), dict(speakers=seed), {}]
    mk = lambda: MultiStreamDiarization(config, 4, gallery=gal)  # noqa: E731
    want = Run(mk(), audios, sched, open_kw).go()
    target = MultiStreamDiarization(config, 4, gallery=gal)
    got = Run(mk(), audios, sched, open_kw, replay=want).go({(5, "after"): [(0, target, dict(gallery=own)), (1, target, None)],
                                               (7, "before"): [(2, None, None)]})
    same(want, got, range(3))
    named = [l for k in range(3) for line in want.rttm[k] for l in line.split() if l.startswith("person")]
    assert named, "some speaker was named"
    # a state named from a gallery needs that gallery
    srv = mk()
    sid = srv.open(gallery=own)
    state = srv.export([sid])[0]
    bare = MultiStreamDiarization(config, 2)
    before = _lib.lib().dg_launch_count()
    with pytest.raises(ValueError, match="gallery"):
        bare.restore([state])
    with pytest.raises(ValueError, match="another gallery"):
        bare.restore([state], gallery=gal)
    assert _lib.lib().dg_launch_count() == before and not bare._open.any()
    assert srv.restore([state], gallery=own) == [sid]


@pytest.mark.parametrize("latency", [0.5, 2.0, 5.0])
def test_vad_continues_exactly(oracle_nets, cuda_device, latency):
    config = vad_config(oracle_nets, cuda_device, latency=latency)
    audios = [synth.synth_audio(S + HOP * 50, seed=600 + k) for k in range(3)]
    sched = schedule(3, TICKS, seed=21)
    mk = lambda: MultiStreamVoiceActivityDetection(config, 4)  # noqa: E731
    want = Run(mk(), audios, sched).go()
    other = MultiStreamVoiceActivityDetection(config, 5, max_windows_per_stream=6)
    got = Run(mk(), audios, sched, replay=want).go({(3, "before"): [(0, other, None)], (5, "after"): [(1, None, None)]})
    same(want, got, range(3))


def test_checkpoints_and_files(oracle_nets, cuda_device, tmp_path):
    """close=False leaves the stream untouched; its checkpoint, saved and loaded, forks an identical continuation"""
    config = make_config(oracle_nets, cuda_device, latency=2.0)
    audios = [synth.synth_audio(S + HOP * 40, seed=700 + k) for k in range(2)]
    sched = schedule(2, TICKS, seed=31)
    mk = lambda: MultiStreamDiarization(config, 3)  # noqa: E731
    want = Run(mk(), audios, sched).go()
    run = Run(mk(), audios, sched, replay=want)
    fork, fork_rttm, n_before = None, [], 0
    for t in range(TICKS):
        p0 = run.pos[0]
        run.push(t)
        if fork is not None and run.pos[0] > p0:
            fork.push(fsid, audios[0][p0:run.pos[0]])
        if t == 6:   # a checkpoint with staged samples
            srv, sid = run.servers[0], run.where[0][1]
            ck = srv.export([sid], close=False)[0]
            ck.save(tmp_path / "ck.npz")
            back = StreamState.load(tmp_path / "ck.npz")
            assert back == ck and back._blob.tobytes() == ck._blob.tobytes()
            assert srv.export([sid], close=False)[0]._blob.tobytes() == ck._blob.tobytes(), "exports are reproducible"
            fork = MultiStreamDiarization(config, 2)
            fsid = fork.restore([back])[0]
            n_before = len(run.rttm.get(0, []))
        run.step()
        if fork is not None:
            fork_rttm += [a.to_rttm() for a in fork.step().get(fsid, [])]
    run.drain(lambda: fork_rttm.extend(a.to_rttm() for a in fork.step().get(fsid, [])))
    same(want, run, range(2))
    assert len(fork_rttm) > 3 and fork_rttm == want.rttm[0][n_before:]


def test_drain_300(oracle_nets, cuda_device):
    config = make_config(oracle_nets, cuda_device, latency=1.0)
    ticks = 4
    base = [synth.synth_audio(S + HOP * 30, seed=800 + i) for i in range(6)]
    audios = [np.ascontiguousarray(base[i % 6][(i // 6) % 20 * HOP:][:S + HOP * 12]) for i in range(300)]
    sched = [[S + HOP if t == 0 else HOP for _ in range(300)] for t in range(ticks * 2)]
    lib = _lib.lib()
    keep = set(range(0, 300, 7))
    want = Run(MultiStreamDiarization(config, 300, max_windows_per_stream=2), audios, sched, keep=keep).go()
    src = MultiStreamDiarization(config, 300, max_windows_per_stream=2)
    run = Run(src, audios, sched, keep=keep, replay=want)
    dst = MultiStreamDiarization(config, 320, max_windows_per_stream=3)
    for t in range(len(sched)):
        run.push(t)
        if t == ticks:
            keys = sorted(run.where)
            before = lib.dg_launch_count()
            states = src.export([run.where[k][1] for k in keys])
            assert lib.dg_launch_count() == before + 1
            before = lib.dg_launch_count()
            sids = dst.restore(states)
            assert lib.dg_launch_count() == before + 1
            run.servers.append(dst)
            for k, s in zip(keys, sids):
                run.where[k] = (1, s)
            assert not src._open.any()
        run.step()
    run.drain()
    same(want, run, sorted(keep))


def test_refusals(oracle_nets, cuda_device):
    config = make_config(oracle_nets, cuda_device, latency=2.0)
    lib = _lib.lib()
    srv = MultiStreamDiarization(config, 3, max_latency=3.0, source_sample_rates=(44100,))
    a = synth.synth_audio(S + HOP * 8, seed=3)
    sid = srv.open(latency=3.0)
    srv.push(sid, a[:S + 2 * HOP])
    srv.step()
    srv.push(sid, a[S + 2 * HOP:S + 6 * HOP])
    st = srv.export([sid], close=False)[0]
    sid44 = srv.open(sample_rate=44100)
    st44 = srv.export([sid44], close=False)[0]
    vsrv = MultiStreamVoiceActivityDetection(vad_config(oracle_nets, cuda_device), 2)
    vad_st = vsrv.export([vsrv.open()])[0]
    seg_o, emb_o = oracle_nets
    nudged = emb_o.state_dict()
    name = next(k for k, v in nudged.items() if v.dtype.is_floating_point and v.numel() > 1)
    nudged[name] = nudged[name].clone()
    nudged[name].view(-1)[0] += 1e-6
    other_models = blocks.SpeakerDiarizationConfig(
        segmentation=config.segmentation, device=cuda_device, latency=2.0,
        embedding=models.EmbeddingModel(models.B200EmbeddingLoader(nudged)))
    cosine_only = make_config(oracle_nets, cuda_device, latency=2.0)
    cosine_only.metric = "euclidean"
    cases = [
        (MultiStreamDiarization(other_models, 2, max_latency=3.0), st, "other models"),
        (MultiStreamDiarization(make_config(oracle_nets, cuda_device, latency=2.0, max_speakers=4), 2, max_latency=3.0),
         st, "settings: max_speakers"),
        (MultiStreamDiarization(make_config(oracle_nets, cuda_device, latency=2.0, beta=9), 2, max_latency=3.0), st,
         "settings: beta"),
        (MultiStreamDiarization(make_config(oracle_nets, cuda_device, latency=2.0, normalize_embedding_weights=True), 2,
                                max_latency=3.0), st, "settings: normalize_embedding_weights"),
        (MultiStreamDiarization(cosine_only, 2, max_latency=3.0), st, "settings: metric"),
        (MultiStreamDiarization(config, 2), st, "max_latency"),
        (MultiStreamDiarization(config, 2, max_latency=3.0), st44, "did not declare"),
        (MultiStreamDiarization(make_config(oracle_nets, cuda_device, latency=2.0, gamma=4), 2, max_latency=3.0), st,
         "settings: gamma"),
        (MultiStreamDiarization(config, 2, max_latency=3.0), vad_st, "vad stream"),
        (MultiStreamVoiceActivityDetection(vad_config(oracle_nets, cuda_device), 2), st, "diarization stream"),
        (MultiStreamDiarization(config, 1, max_windows_per_stream=1, max_latency=3.0), st, "capacity"),
    ]
    for target, state, words in cases:
        before = lib.dg_launch_count()
        with pytest.raises(ValueError, match=words):
            target.restore([state])
        assert lib.dg_launch_count() == before and not target._open.any()
    full = MultiStreamDiarization(config, 1, max_latency=3.0)
    full.open()
    with pytest.raises(ValueError, match="free slots"):
        full.restore([st])
    bad = StreamState(st._blob, dict(st._meta, version=99))
    with pytest.raises(ValueError, match="format version"):
        MultiStreamDiarization(config, 2, max_latency=3.0).restore([bad])


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two visible GPUs")
def test_move_to_another_gpu(oracle_nets):
    d0, d1 = torch.device("cuda", 0), torch.device("cuda", 1)
    audios = [synth.synth_audio(S + HOP * 30, seed=900)]
    sched = schedule(1, 10, seed=1)
    want = Run(MultiStreamDiarization(make_config(oracle_nets, d0, latency=1.0), 2), audios, sched).go()
    other = MultiStreamDiarization(make_config(oracle_nets, d1, latency=1.0), 2)
    got = Run(MultiStreamDiarization(make_config(oracle_nets, d0, latency=1.0), 2), audios, sched, replay=want).go(
        {(4, "after"): [(0, other, None)]})
    same(want, got, [0])
