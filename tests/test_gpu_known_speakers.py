"""Known speakers on the device (diart_b200.speakers): a pipeline or a live stream seeded with known centroids is the
reference's clustering on a pre-filled state -- the float64 oracle seeded the same way and replayed on the device's own
scores and embeddings gives its speaker maps and centroids bit for bit -- its annotations name the known speakers, a
stream exported with speakers() resumes exactly, and enroll() computes each clip's centroid from one sweep.

Models and audio are the seeded synthetic ones of diart_b200.synth."""
import ctypes as C
import math

import numpy as np
import pytest
import torch

from diart_b200 import _lib, blocks, models, synth
from diart_b200.core import SlidingWindow, SlidingWindowFeature
from diart_b200.serve import MultiStreamDiarization, MultiStreamVoiceActivityDetection
from diart_b200.speakers import KnownSpeakers, dominant_speaker, enroll, exported, speaker_labels
from diart_b200.tune import DatasetSweep
from oracle.clustering import OracleClustering
from test_gpu_multi_stream import EMB_TOL, Recorder
from test_gpu_multi_stream_config import README_ROWS, diarization_variant, run_ragged, values
from test_gpu_multi_stream_vad import make_config as make_vad_config

pytestmark = pytest.mark.gpu

SR, S, HOP = 16000, 80000, 8000
NAMES = ("alice", "bob", "carol")


@pytest.fixture(scope="module")
def states():
    return synth.segmentation_state(), synth.embedding_state()


def make_config(states, device, **kw):
    seg_state, emb_state = states
    return blocks.SpeakerDiarizationConfig(
        segmentation=models.SegmentationModel(models.B200SegmentationLoader(seg_state)),
        embedding=models.EmbeddingModel(models.B200EmbeddingLoader(emb_state)), device=device, **kw)


def window(audio, i):
    return SlidingWindowFeature(audio[i * HOP:i * HOP + S, None], SlidingWindow(start=i * 0.5, duration=1 / SR, step=1 / SR))


def device_window(audio, i, device):
    return torch.from_numpy(synth.windows(audio, 1, first=i)).to(device)


def learned(config, seed, names, windows=14):
    """known speakers with realistic centroids: the first len(names) centres a fresh pipeline holds after ``windows``
    windows of a 4-speaker stream, renamed"""
    pipe = blocks.SpeakerDiarization(config)
    audio = synth.synth_audio(S + HOP * windows, seed=seed)
    for i in range(windows):
        pipe.device_step(device_window(audio, i, config.device))
    state = pipe.speakers()
    assert len(state) >= len(names), f"only {len(state)} speakers after {windows} windows"
    return KnownSpeakers(names, state.centroids[:len(names)])


def seeded_oracle(config, known, **kw):
    p = dict(tau_active=config.tau_active, rho_update=config.rho_update, delta_new=config.delta_new)
    p.update({k: v for k, v in kw.items() if v is not None and k in p})
    clu = OracleClustering(p["tau_active"], p["rho_update"], p["delta_new"], "cosine", config.max_speakers)
    if known is not None and len(known):
        clu.centers = np.zeros((config.max_speakers, known.dimension))
        clu.centers[:len(known)] = known.centroids
        clu.active_centers = set(range(len(known)))
    return clu


def oracle_state(clu, labels):
    """the oracle's state as speakers() exports it"""
    if clu.centers is None:
        return KnownSpeakers([], np.zeros((0, 0)))
    return exported(labels, clu.centers, [int(g in clu.active_centers) for g in range(clu.max_speakers)])


def same_state(a, b):
    return a.names == b.names and len(a) == len(b) and (
        len(a) == 0 or np.array_equal(a.centroids.view(np.int64), b.centroids.view(np.int64)))


def run_pipeline(config, known, audio, first, last, shift=0.0):
    """a seeded pipeline fed windows first .. last - 1 one per call, and a twin in the same state -> (annotations, scores,
    embeddings, maps of the twin's fused steps, the two pipelines)"""
    pipe, twin = blocks.SpeakerDiarization(config), blocks.SpeakerDiarization(config)
    for p in (pipe, twin):
        p.set_known_speakers(known)
        p.set_timestamp_shift(shift)
    anns, seg, emb, maps = [], [], [], []
    for i in range(first, last):
        anns.append(pipe([window(audio, i)])[0][0])
        s, e, m = twin.device_step(device_window(audio, i, config.device))
        seg.append(s.cpu().numpy()[0]), emb.append(e.cpu().numpy()[0]), maps.append(m.cpu().numpy()[0])
    return anns, np.stack(seg), np.stack(emb), np.stack(maps), pipe, twin


def check_labels(anns, maps, labels, n_known):
    """every turn of window i is labelled labels[g] for a global speaker g some window up to i was mapped to; a known one
    (g < n_known) carries its name, never speaker<g>"""
    seen, named = set(), 0
    index = {label: g for g, label in enumerate(labels)}
    for ann, m in zip(anns, maps):
        seen |= {int(g) for g in m if g >= 0}
        for _, _, label in ann.itertracks(yield_label=True):
            assert label in index, label
            assert index[label] in seen, (label, sorted(seen))
            named += index[label] < n_known
    assert all(f"speaker{g}" not in index for g in range(n_known))
    return named


def test_a_seeded_pipeline_is_the_oracle_on_a_prefilled_state(states, cuda_device):
    config = make_config(states, cuda_device, latency=2.0)
    known = learned(config, 2101, NAMES)
    audio = synth.synth_audio(S + HOP * 30, seed=2102)
    anns, seg, emb, maps, pipe, twin = run_pipeline(config, known, audio, 0, 30)
    clu = seeded_oracle(config, known)
    want = np.stack([clu(s, e)[0] for s, e in zip(seg, emb)])
    assert np.array_equal(maps, want)
    labels = speaker_labels(known, config.max_speakers)
    final = oracle_state(clu, labels)
    assert len(final) > len(known), "no speaker was discovered besides the known ones"
    assert same_state(twin.speakers(), final) and same_state(pipe.speakers(), final)
    assert final.names[:3] == NAMES
    assert check_labels(anns, maps, labels, len(known)) > 0, "no turn of a known speaker"
    # reset() re-applies the known speakers: the same input gives the same output
    rttm = [a.to_rttm() for a in anns]
    pipe.reset()
    twin.reset()
    assert same_state(pipe.speakers(), known)
    again = [pipe([window(audio, i)])[0][0].to_rttm() for i in range(30)]
    again_maps = np.stack([twin.device_step(device_window(audio, i, cuda_device))[2].cpu().numpy()[0] for i in range(30)])
    assert again == rttm and np.array_equal(again_maps, maps)
    # only before the first chunk
    for p in (pipe, twin):
        with pytest.raises(ValueError, match="before the first chunk"):
            p.set_known_speakers(known)
    pipe.reset()
    pipe.set_known_speakers(None)                     # allowed again, and back to the fresh state
    fresh = blocks.SpeakerDiarization(config)
    assert [pipe([window(audio, i)])[0][0].to_rttm() for i in range(6)] == \
        [fresh([window(audio, i)])[0][0].to_rttm() for i in range(6)]


def test_known_speakers_of_another_dimension_are_refused_before_any_launch(states, cuda_device):
    config = make_config(states, cuda_device)
    audio = synth.synth_audio(S, seed=3)
    blocks.SpeakerDiarization(config)([window(audio, 0)])          # loads the models
    pipe = blocks.SpeakerDiarization(config)
    pipe.set_known_speakers(KnownSpeakers(["alice"], np.ones((1, 16))))
    lib = _lib.lib()
    before = lib.dg_launch_count()
    with pytest.raises(ValueError, match="dimension 16"):
        pipe([window(audio, 0)])
    assert lib.dg_launch_count() == before
    with pytest.raises(ValueError, match="at most max_speakers"):
        blocks.SpeakerDiarization(config).set_known_speakers(
            KnownSpeakers([f"n{i}" for i in range(21)], np.ones((21, 512))))


def test_the_blockwise_path_names_the_known_speakers(states, oracle_nets, cuda_device):
    """foreign models (torch modules behind the loader API) run block by block; Binarize labels the turns"""
    import copy

    native = make_config(states, cuda_device)
    known = learned(native, 2101, NAMES)
    seg_o, emb_o = (copy.deepcopy(m) for m in oracle_nets)
    config = blocks.SpeakerDiarizationConfig(segmentation=models.SegmentationModel(lambda: seg_o),
                                             embedding=models.EmbeddingModel(lambda: emb_o), device=cuda_device,
                                             latency=1.0)
    pipe = blocks.SpeakerDiarization(config)
    pipe.set_known_speakers(known)
    audio = synth.synth_audio(S + HOP * 12, seed=2102)
    anns = [pipe([window(audio, i)])[0][0] for i in range(12)]
    state = pipe.speakers()
    assert state.names[:3] == NAMES
    labels = speaker_labels(known, config.max_speakers)
    used = {label for a in anns for _, _, label in a.itertracks(yield_label=True)}
    assert used and used <= set(labels[:len(state)]) and used & set(NAMES)


@pytest.mark.parametrize("latency", [0.5, 2.5])
def test_a_pipeline_resumes_from_an_exported_state(states, cuda_device, latency):
    config = make_config(states, cuda_device, latency=latency)
    known = learned(config, 2201, NAMES[:2])
    N, n, shift = 32, 13, 1.25
    audio = synth.synth_audio(S + HOP * N, seed=2202)
    a_pipe, a_twin = blocks.SpeakerDiarization(config), blocks.SpeakerDiarization(config)
    for p in (a_pipe, a_twin):
        p.set_known_speakers(known)
        p.set_timestamp_shift(shift)
    a_rttm, a_maps, snapshot = [], [], None
    for i in range(N):
        if i == n:
            snapshot = a_pipe.speakers()
            assert same_state(snapshot, a_twin.speakers()) and len(snapshot) > len(known)
        a_rttm.append(a_pipe([window(audio, i)])[0][0].to_rttm())
        a_maps.append(a_twin.device_step(device_window(audio, i, cuda_device))[2].cpu().numpy()[0])
    anns, _, _, b_maps, b_pipe, b_twin = run_pipeline(config, snapshot, audio, n, N, shift)
    assert np.array_equal(b_maps, np.stack(a_maps[n:]))
    lag = int(round(latency / config.step)) - 1       # outputs that aggregate fewer buffers after the resume
    b_rttm = [a.to_rttm() for a in anns]
    assert b_rttm[lag:] == a_rttm[n + lag:]
    assert same_state(b_pipe.speakers(), a_pipe.speakers())
    assert any(known.names[0] in r or known.names[1] in r for r in b_rttm)


def dedicated_seeded(config, known, audio, n, shift=0.0):
    """a SpeakerDiarization with set_known_speakers(known) fed one window per call -> (RTTM per window, scores,
    embeddings, maps)"""
    anns, seg, emb, maps, _, _ = run_pipeline(config, known, audio, 0, n, shift)
    return [a.to_rttm() for a in anns], seg, emb, maps


class StateRecorder(Recorder):
    """a Recorder that checks, after every tick, each open stream's speakers() against the oracle seeded with its known
    speakers and replayed on its scores and embeddings of the tick outputs"""

    def __init__(self, server, plan):
        super().__init__(server)
        self.plan, self.oracles, self.done, self.checked = plan, {}, {}, 0

    def tick(self):
        got = super().tick()
        server = self.server
        for sid in np.flatnonzero(server._open).tolist():
            k = self.sid_key[sid]
            kw = self.plan[k][3]
            known = kw.get("speakers")
            if k not in self.oracles:
                self.oracles[k] = seeded_oracle(server.config, known, **kw)
                self.done[k] = 0
            clu, d = self.oracles[k], self.done[k]
            seg, emb, maps = self.seg.get(k, []), self.emb.get(k, []), self.maps.get(k, [])
            for i in range(d, len(seg)):
                assert np.array_equal(clu(seg[i], emb[i])[0], maps[i]), f"stream {k}: map {i}"
            self.done[k] = len(seg)
            labels = speaker_labels(known if known is not None and len(known) else None, server.config.max_speakers)
            assert same_state(server.speakers(sid), oracle_state(clu, labels)), f"stream {k}: state"
            self.checked += 1
        return got


def test_seeded_and_unseeded_streams_on_one_server(states, cuda_device):
    config = make_config(states, cuda_device, latency=1.0)
    three, two = learned(config, 2301, NAMES), learned(config, 2302, ("dan", "speaker1"))
    rows = [values(r) for r in README_ROWS]
    # (windows, when, shift, open kwargs): seeded streams 0, 2, 5 and 7 (7 reopens stream 4's slot, 4 seeded with
    # nothing), the others unseeded
    plan = [(24, 0, 0.0, dict(latency=2.0, speakers=three, **rows[0])),
            (22, 0, 1.5, dict(latency=0.5, **rows[1])),
            (20, 1, 0.0, dict(speakers=two)),
            (26, 0, 0.0, dict(latency=5.0, **rows[3])),
            (9, 0, 0.0, dict(latency=0.5, speakers=KnownSpeakers([], []))),
            (18, 2, 2.0, dict(latency=5.0, speakers=three, **rows[2])),
            (16, 1, 0.0, dict()),
            (15, ("after", 4), 0.0, dict(latency=2.0, speakers=two, **rows[1]))]
    audio = {k: synth.synth_audio(S + HOP * (n + 5), seed=2310 + k) for k, (n, _, _, _) in enumerate(plan)}
    seeded = [k for k, p in enumerate(plan) if len(p[3].get("speakers") or ())]
    assert seeded == [0, 2, 5, 7]

    def run(plan):
        server = MultiStreamDiarization(config, max_streams=7, max_windows_per_stream=4, max_latency=5.0)
        rec = StateRecorder(server, plan)
        per_tick, reused = run_ragged(server, rec, audio, plan, np.random.default_rng(41), lambda r, k: len(r.rttm.get(k, [])))
        return rec, per_tick, reused

    rec, per_tick, reused = run(plan)
    assert [k for k, _, _ in reused] == [7] and reused[0][1] in reused[0][2]
    assert rec.checked > 3 * len(per_tick)
    for k in seeded:
        n, _, shift, kw = plan[k]
        kw = dict(kw)
        known = kw.pop("speakers")
        rttm, seg, emb, maps = dedicated_seeded(diarization_variant(config, **kw), known, audio[k], n, shift)
        assert rec.rttm[k][:n] == rttm, f"stream {k}: RTTM differs"
        assert np.array_equal(np.stack(rec.seg[k][:n]), seg), f"stream {k}: scores differ"
        assert np.abs(np.stack(rec.emb[k][:n]) - emb).max() <= EMB_TOL, f"stream {k}: embeddings differ"
        assert np.array_equal(np.stack(rec.maps[k][:n]), maps), f"stream {k}: speaker maps differ"
        assert any(name in line for r in rttm for line in r.splitlines() for name in known.names if not
                   name.startswith("speaker")), f"stream {k}: no turn of a known speaker"
    # the unseeded streams give what they give when no stream is seeded
    plain = [(n, when, shift, {key: v for key, v in kw.items() if key != "speakers"}) for n, when, shift, kw in plan]
    base, base_ticks, _ = run(plain)
    assert base_ticks == per_tick
    for k in range(len(plan)):
        if k in seeded:
            continue
        for name in ("rttm", "seg", "emb", "maps"):
            want, got = getattr(base, name)[k], getattr(rec, name)[k]
            assert len(got) == len(want)
            if name == "rttm":
                assert got == want, f"stream {k}: RTTM"
            else:
                assert np.array_equal(np.stack(got), np.stack(want)), f"stream {k}: {name}"


def test_seeded_refusals_leave_the_slot_closed(states, cuda_device):
    config = make_config(states, cuda_device, max_speakers=4)
    server = MultiStreamDiarization(config, max_streams=2, max_windows_per_stream=2)
    lib = _lib.lib()
    before = lib.dg_launch_count()
    good = np.ones((2, server.D))
    for make in (lambda: KnownSpeakers(["a", "b"], np.ones((2, 16))),                       # wrong dimension
                 lambda: KnownSpeakers([f"n{i}" for i in range(5)], np.ones((5, server.D))),  # more than max_speakers
                 lambda: KnownSpeakers(["a", "b"], np.r_[good[:1], np.zeros((1, server.D))]),
                 lambda: KnownSpeakers(["a", "b"], np.r_[good[:1], np.full((1, server.D), math.nan)]),
                 lambda: KnownSpeakers(["a", "b c"], good),
                 lambda: KnownSpeakers(["speaker1", "b"], good)):
        with pytest.raises(ValueError):
            server.open(speakers=make())
    params = np.array([0.5, 0.3, 1.0])
    bad_rows = np.ones((5, server.D))
    zero = np.r_[good[:1], np.zeros((1, server.D))]
    nan = np.r_[good[:1], np.full((1, server.D), math.inf)]
    for table, n in ((bad_rows, 5), (good, -1), (zero, 2), (nan, 2), (None, 2)):
        ptr = None if table is None else np.ascontiguousarray(table).ctypes.data
        assert lib.dg_multi_open_seeded(server.handle, 0, -1, 1, params.ctypes.data, ptr, n) == -1
        assert b"dg_multi_open_seeded" in lib.dg_last_error()
    assert lib.dg_multi_open_seeded(server.handle, 0, -1, server.nw + 1, params.ctypes.data, good.ctypes.data, 2) == -1
    vad = MultiStreamVoiceActivityDetection(make_vad_config(states[0], cuda_device), 2)
    for n in (0, 1):
        assert lib.dg_multi_open_seeded(vad.handle, 0, -1, 1, params.ctypes.data, good.ctypes.data, n) == -1
        assert b"dg_multi_open_seeded" in lib.dg_last_error()
    state = np.empty((4, server.D)), np.empty(4, dtype=np.int32), C.c_int()
    assert lib.dg_multi_get_state(server.handle, 0, state[0].ctypes.data, state[1].ctypes.data, C.byref(state[2])) == -1
    assert lib.dg_launch_count() == before
    for s in (server, vad):
        assert not s._open.any()
        for slot in (0, 1):
            assert lib.dg_multi_available(s.handle, slot) == -1
    # still usable: a seeded stream opens in slot 0, and exports its seed before its first tick
    known = KnownSpeakers(["a", "b"], np.stack([np.r_[1.0, np.zeros(server.D - 1)], np.r_[0.0, 1.0, np.zeros(server.D - 2)]]))
    sid = server.open(speakers=known)
    assert sid == 0 and same_state(server.speakers(sid), known)


def one_speaker(seconds, seed):
    return synth.synth_audio(int(seconds * SR), seed=seed, num_speakers=1)


def test_enrollment_is_the_dominant_speakers_final_centroid(states, cuda_device):
    config = make_config(states, cuda_device, latency=1.0)
    clips = [("alice", one_speaker(12, 2401)), ("bob", one_speaker(8.5, 2402)), ("carol", one_speaker(3, 2403)),
             ("dan", one_speaker(20, 2404))]
    known = enroll(config, clips)
    assert known.names == ("alice", "bob", "carol", "dan")
    ds = DatasetSweep(config, [(name, wav, None) for name, wav in clips])
    assert ds.offsets[3] - ds.offsets[2] == 1          # carol's 3 s clip is one left-padded window
    predictions = ds.run([{}])
    labels = speaker_labels(None, config.max_speakers)
    for f, (name, _) in enumerate(clips):
        g = dominant_speaker(predictions[f][0], labels)
        assert g is not None, f"{name}: no speech in the prediction, the comparison says little"
        seg, emb = (t.cpu().numpy() for t in ds.file_outputs(f))
        clu = seeded_oracle(config, None)
        for s, e in zip(seg, emb):
            clu(s, e)
        assert np.array_equal(known.centroids[f].view(np.int64), clu.centers[g].view(np.int64)), name
    # a clip whose prediction has no speech names the clip: a 7 kHz tone of whole steps scores below tau_active in every
    # frame, at latency 0.5 (no right padding: silence scores above it)
    t = np.arange(8 * SR) / SR
    tone = (0.9 * np.sin(2 * np.pi * 7000 * t)).astype(np.float32)
    quiet = make_config(states, cuda_device)
    silent = DatasetSweep(quiet, [("tone", tone, None)])
    assert silent.seg.max().item() < quiet.tau_active
    with pytest.raises(ValueError, match="clip 'tone'"):
        enroll(quiet, [clips[3], ("tone", tone)])
    # enrolled speakers seed a stream
    server = MultiStreamDiarization(config, max_streams=2)
    sid = server.open(speakers=known)
    audio = synth.synth_audio(S + HOP * 6, seed=2405)
    server.push(sid, audio)
    out = []
    while server.available(sid):
        out += server.step()[sid]
    assert len(out) == 7
    assert server.speakers(sid).names[:4] == known.names
