"""Moving live streams, host side: dg_multi_export / dg_multi_import piece plans against a numpy model of the rings (through
the host-only hook dg_selftest_multi_transfer_host, where the pieces run on the host), the refusals that need no device,
and StreamState's .npz."""
import ctypes as C

import numpy as np
import pytest

from diart_b200 import _lib
from diart_b200.transfer import VERSION, StreamState

# pipeline windows of 800 / 80 samples; a declared rate resampled 3 -> 2 (half-width 2) with windows of 1200 / 120 source
# samples: 16 kHz frames 1 .. 398 of a window are interior, 40 frames per step
OUT_CHUNK, OUT_STEP, F = 800, 80, 5
RATE = (3, 2, 2, 1200, 120)


def ring_capacity(S, hop, max_wps):
    return (S + 2 * max_wps * hop + 1023) // 1024 * 1024


def run(ops, src_slot, patch=0, src=(3, 2, 4), dst=(2, 8, 6)):
    """drives a source VAD handle (slots, max_wps, nw) with ops, exports src_slot and imports it into a target ->
    (results, info dict, target ring, frame ring, history, message, the samples pushed per op)"""
    lib = _lib.lib()
    geom = np.array([src[0], src[1], src[2], OUT_CHUNK, OUT_STEP, F, *RATE, *dst], dtype=np.int32)
    ops = np.ascontiguousarray(ops, dtype=np.int32).reshape(-1, 3)
    total = int(ops[ops[:, 0] == 2, 2].sum())
    samples = np.arange(1, total + 1, dtype=np.float32)
    result = np.empty(len(ops), np.int32)
    cap = 1 << 16
    ring, yring, hist = (np.zeros(cap, np.float32) for _ in range(3))
    info = np.zeros(16, np.int64)
    msg = C.create_string_buffer(512)
    rc = lib.dg_selftest_multi_transfer_host(geom.ctypes.data, len(ops), ops.ctypes.data, samples.ctypes.data,
                                             result.ctypes.data, src_slot, patch, ring.ctypes.data, yring.ctypes.data,
                                             hist.ctypes.data, cap, info.ctypes.data, msg, len(msg))
    assert rc == 0, lib.dg_last_error().decode()
    keys = ["rc", "C", "Q", "Y", "wpos", "rpos", "done", "n_hist", "frame0", "n_frames", "bytes", "src_C", "src_Q"]
    return result, dict(zip(keys, info.tolist())), ring, yring, hist, msg.value.decode(), samples


def script(rng, n_ticks=40, close_at=12):
    """stream A (slot 0, resampled) and stream B (slot 1, pipeline rate) push ragged blocks interleaved with a third stream
    (slot 2) that is closed with staged samples and reopened; the last pushes of A and B stay staged.  -> (ops, the sample
    ranges of each op's push, per slot)"""
    ops = [(0, 0, 0), (0, 1, -1), (0, 2, -1)]
    for t in range(n_ticks + 1):
        for slot, lo, hi in ((0, 30, 400), (2, 5, 200), (1, 10, 160), (0, 1, 50)):
            ops.append((2, slot, int(rng.integers(lo, hi))))
        if t == close_at:
            ops += [(1, 2, 0), (0, 2, -1), (2, 2, 33)]
        if t < n_ticks:
            ops.append((4, 0, 0))
    return ops


def stream_samples(ops, result, samples, slot):
    """the samples of the stream in `slot` at the end, in stream order (pushes the source accepted since its last open)"""
    out, pos = [], 0
    for (kind, s, n), rc in zip(ops, result):
        if kind == 0 and s == slot:
            out = []
        if kind == 2 and rc == 0 and n > 0:
            if s == slot:
                out.append(samples[pos:pos + n])
            pos += n
    return np.concatenate(out)


@pytest.mark.parametrize("src,dst", [((3, 2, 4), (2, 8, 6)), ((3, 8, 6), (1, 2, 6)), ((3, 2, 4), (3, 2, 4))],
                         ids=["to-larger", "to-smaller", "same"])
def test_resampled_stream_moves_exactly(src, dst):
    """ring wrap-around on both sides, capacities and frame rings that differ, history re-strided across nw, staged pieces
    interleaved with other streams' pushes and a close"""
    rng = np.random.default_rng(3)
    ops = script(rng)
    result, info, ring, yring, hist, msg, samples = run(ops, 0, src=src, dst=dst)
    assert info["rc"] == 0, msg
    want = stream_samples(ops, result, samples, 0)
    o, n, w, chunk, step = RATE
    wpos, rpos, C_t, Q_t = info["wpos"], info["rpos"], info["C"], info["Q"]
    assert wpos == len(want) and rpos % step == 0 and wpos - rpos > 0
    assert wpos > info["src_C"] and wpos > C_t, "the positions wrap both rings"
    assert C_t == ring_capacity(chunk, step, dst[1]) and info["src_C"] == ring_capacity(chunk, step, src[1])
    pos = np.arange(rpos, wpos)
    assert np.array_equal(ring[pos % C_t], want[rpos:wpos]), "audio [rpos, wpos) at absolute position mod C"
    # the frames a future window still reads: [rpos / o + r_lo, done), at frame R mod Q
    assert info["frame0"] == rpos // o + 1 and info["n_frames"] == info["done"] - info["frame0"] > 0
    R = np.arange(info["frame0"], info["done"])
    got = yring[((R % Q_t)[:, None] * n + np.arange(n)[None, :])]
    assert np.array_equal(got, (R[:, None] * n + np.arange(n)[None, :]).astype(np.float32))
    # history: the last n_hist chunks, oldest first, at the target's stride
    nh = info["n_hist"]
    assert nh == src[2] - 1
    c0 = rpos // step - nh
    want_hist = ((c0 + np.arange(nh))[:, None] * F + np.arange(F)[None, :]).astype(np.float32)
    assert np.array_equal(hist[:nh * F].reshape(nh, F), want_hist)
    assert info["bytes"] % 16 == 0


def test_stream_at_the_pipeline_rate_moves_exactly():
    rng = np.random.default_rng(4)
    ops = script(rng, n_ticks=25)
    result, info, ring, yring, hist, msg, samples = run(ops, 1)
    assert info["rc"] == 0, msg
    want = stream_samples(ops, result, samples, 1)
    pos = np.arange(info["rpos"], info["wpos"])
    assert np.array_equal(ring[pos % info["C"]], want[info["rpos"]:])
    assert info["n_frames"] == 0 and info["done"] == 0


def test_a_stream_before_its_first_window():
    """everything staged, nothing ticked: the audio is all staged samples, no frames, no history"""
    ops = [(0, 0, 0), (2, 0, 500), (0, 1, -1), (2, 1, 7), (2, 0, 300)]
    result, info, ring, yring, hist, msg, samples = run(ops, 0)
    assert info["rc"] == 0 and info["rpos"] == 0 and info["wpos"] == 800 and info["n_hist"] == 0
    assert info["n_frames"] == 0
    want = np.concatenate([samples[:500], samples[507:807]])
    assert np.array_equal(ring[:800], want)


@pytest.mark.parametrize("patch,words", [(1, "format version"), (2, "diarization stream"), (3, "windows of"),
                                         (4, "max_latency"), (5, "capacity"), (6, "failed on its source"),
                                         (7, "did not declare"), (8, "not a packed stream state")])
def test_import_refusals(patch, words):
    rng = np.random.default_rng(5)
    _, info, *_, msg, _ = run(script(rng, n_ticks=6), 0, patch=patch)
    assert info["rc"] == -1
    assert msg.startswith("dg_multi_import: state 0") and words in msg, msg


def test_entry_points_refuse_bad_arguments():
    lib = _lib.lib()
    slots = np.zeros(1, np.int32)
    sizes = np.zeros(1, np.int64)
    out = np.zeros(16, np.uint8)
    assert lib.dg_multi_export_bytes(None, slots.ctypes.data, 1, sizes.ctypes.data) == -1
    assert "dg_multi_export_bytes" in lib.dg_last_error().decode()
    assert lib.dg_multi_export(None, slots.ctypes.data, 1, 1, out.ctypes.data, 16) == -1
    assert "dg_multi_export" in lib.dg_last_error().decode()
    assert lib.dg_multi_import(None, out.ctypes.data, 16, 1, None, slots.ctypes.data) == -1
    assert "dg_multi_import" in lib.dg_last_error().decode()


def test_stream_state_save_load(tmp_path):
    blob = np.random.default_rng(0).integers(0, 256, 4096).astype(np.uint8)
    meta = dict(version=VERSION, kind="vad", rate=44100, latency=2.0, shift=1.5, labels=["a", "speaker1"], gallery=None)
    st = StreamState(blob, meta)
    st.save(tmp_path / "s.npz")
    back = StreamState.load(tmp_path / "s.npz")
    assert back == st and back._blob.tobytes() == blob.tobytes()
    assert (back.kind, back.sample_rate, back.latency, back.nbytes) == ("vad", 44100, 2.0, 4096)
    np.savez(tmp_path / "v2.npz", version=np.int64(VERSION + 1), blob=blob, meta=np.zeros(2, np.uint8))
    with pytest.raises(ValueError, match="format version"):
        StreamState.load(tmp_path / "v2.npz")
    np.savez(tmp_path / "other.npz", x=np.zeros(3))
    with pytest.raises(ValueError, match="not a saved stream state"):
        StreamState.load(tmp_path / "other.npz")


def test_import_refusal_of_a_failed_clustering_is_a_value_error():
    """a packed state whose clustering failed on its source is refused like every other bad state: ValueError, not the
    AssertionError that exporting such a stream raises"""
    rng = np.random.default_rng(5)
    _, info, *_, msg, _ = run(script(rng, n_ticks=6), 0, patch=6)
    assert info["rc"] == -1 and "Cannot update unknown centers" not in msg
    with pytest.raises(ValueError, match="failed on its source"):   # the refusal as restore reports it
        _lib.check(info["rc"])


def test_model_fingerprints(oracle_nets):
    from diart_b200 import models
    from diart_b200.transfer import model_fingerprint

    seg_o, emb_o = oracle_nets
    sd = seg_o.state_dict()
    a, b = models.B200PyanNet(sd), models.B200PyanNet(dict(sd))
    assert model_fingerprint(a) == model_fingerprint(b), "the same weights in another object"
    name = next(k for k, v in sd.items() if v.dtype.is_floating_point and v.numel() > 1)
    nudged = dict(sd)
    nudged[name] = sd[name].clone()
    nudged[name].view(-1)[0] += 1e-6
    assert model_fingerprint(models.B200PyanNet(nudged)) != model_fingerprint(a), "one weight off by 1e-6"
    assert model_fingerprint(models.B200PyanNet(sd, powerset=(3, 2))) != model_fingerprint(a), "a powerset head"
    esd = emb_o.state_dict()
    e31, e21 = models.B200XVectorSincNet(esd, "3.1"), models.B200XVectorSincNet(esd, "2.1")
    assert model_fingerprint(e31) != model_fingerprint(e21), "another pool_mode"
    assert model_fingerprint(e31) != model_fingerprint(a)


def test_gallery_fingerprints():
    from diart_b200.speakers import KnownSpeakers, SpeakerGallery
    from diart_b200.transfer import gallery_fingerprint

    rng = np.random.default_rng(1)
    rows = rng.standard_normal((4, 16))
    fp = lambda names, c, thr=0.5: gallery_fingerprint(SpeakerGallery(KnownSpeakers(names, c), thr, "cuda"))  # noqa: E731
    base = fp(["a", "b", "c", "d"], rows)
    assert fp(["a", "b", "c", "d"], rows.copy(), thr=0.9) == base, "the threshold stays with each stream"
    assert fp(["a", "b", "c", "e"], rows) != base
    moved = rows.copy()
    moved[2, 3] += 1e-9
    assert fp(["a", "b", "c", "d"], moved) != base
    assert fp(["a", "b", "d", "c"], rows[[0, 1, 3, 2]]) != base, "entry order is part of the gallery"
