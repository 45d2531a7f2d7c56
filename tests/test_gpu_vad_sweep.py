"""VAD sweep on the device (dg_vad_sweep_* through diart_b200.tune.VoiceActivitySweep): the resident scores are the
segmentation's bits, every (file, trial) prediction equals a VoiceActivityDetection run with that tau_active, the per-chunk
turns equal the device post-path's, the detection error components equal oracle/detection.py bit for bit, results do not
depend on the other trials or files, scoring runs no network kernel and bad arguments never launch."""
import ctypes

import numpy as np
import pytest
import torch

from diart_b200 import _lib, blocks, models, synth
from diart_b200.blocks.post import DevicePostPath
from diart_b200.core import SlidingWindow, SlidingWindowFeature
from diart_b200.sinks import PredictionAccumulator
from diart_b200.tune import PATCH_COLLAR, VoiceActivitySweep, file_windows, seg_resolution
from oracle.detection import detection_components
from test_gpu_sweep_score import synth_reference

pytestmark = pytest.mark.gpu

# as test_gpu_sweep_dataset: one window with left padding, 256, 257 and 601 windows, two others
SECONDS = (3.2, 132.3, 132.8, 304.7, 61.3, 47.9)
TAUS = [None, 0.0, 1.0, 0.3, 0.45, 0.55, 0.7, 0.85]      # None: the config's value


def make_config(oracle_nets, device, **kw):
    seg_o, _ = oracle_nets
    return blocks.VoiceActivityDetectionConfig(
        segmentation=models.SegmentationModel(models.B200SegmentationLoader(seg_o.state_dict())), device=device, **kw)


def make_files():
    files = []
    for i, secs in enumerate(SECONDS):
        x = synth.synth_audio(int(secs * 16000), seed=900 + i, num_speakers=3 + i % 3)
        files.append((f"file{i}", x, synth_reference(60 + i, 3 + i % 4, secs, uri=f"file{i}")))
    return files


def as_trials(taus):
    return [{} if t is None else {"tau_active": t} for t in taus]


def pipeline_prediction(config, fw, uri, tau):
    """Benchmark.run_single with VoiceActivityDetection(config, tau_active=tau) over the sweep's windows, batches of 256"""
    config.tau_active = tau
    pipe = blocks.VoiceActivityDetection(config)
    pipe.set_timestamp_shift(-fw.padding[0])
    acc = PredictionAccumulator(uri)
    sr = config.sample_rate
    chunks = [SlidingWindowFeature(fw.window(i)[:, None], SlidingWindow(start=fw.starts[i], duration=1 / sr, step=1 / sr))
              for i in range(fw.num_windows)]
    for i in range(0, len(chunks), 256):
        for out in pipe(chunks[i:i + 256]):
            acc.on_next(out)
    return acc.get_prediction()


def equal_to_a_curve_value(vs, f, c, fa):
    """the aggregated curve value of frame fa of chunk c (file f) at latency = step (one buffer): h * v / h in float64"""
    c0 = int(vs.offsets[f])
    nb, lo = int(vs.plan[c0 + c, 0]), int(vs.plan[c0 + c, 4])
    assert nb == 1 and vs.plan[c0 + c, 2] == 0
    F = vs.seg.shape[1]
    idx = min(max(lo + fa, 0), F - 1)
    v = float(vs.seg[c0 + c, idx].amax().item())
    h = np.hamming(F)[idx]
    return (h * v) / h


@pytest.fixture(scope="module")
def dataset(oracle_nets, cuda_device):
    cfg = make_config(oracle_nets, cuda_device)
    files = make_files()
    vs = VoiceActivitySweep(cfg, files)
    taus = TAUS + [equal_to_a_curve_value(vs, 1, 7, 11), equal_to_a_curve_value(vs, 3, 300, 4)]
    return cfg, files, vs, as_trials(taus)


def test_windows_of_the_chosen_lengths(oracle_nets, cuda_device):
    cfg = make_config(oracle_nets, cuda_device)
    fws = [file_windows(np.zeros(int(s * 16000), np.float32), cfg) for s in SECONDS]
    assert [fw.num_windows for fw in fws[:4]] == [1, 256, 257, 601]
    assert fws[0].padding[0] > 0 and all(fw.padding[0] == 0 for fw in fws[1:])


def test_resident_scores_equal_forward_device(dataset):
    cfg, files, vs, _ = dataset
    N, F, K = vs.seg.shape
    assert vs.num_chunks == N == sum(file_windows(x, cfg).num_windows for _, x, _ in files)
    assert vs.resident_bytes == N * F * K * 4 + vs.curve_frames * 8
    seg = vs.pipeline.segmentation
    for f, (_, x, _) in enumerate(files):
        fw = file_windows(x, cfg)
        stacked = np.stack([fw.window(i) for i in range(fw.num_windows)])
        want = torch.cat([seg.forward_device(torch.from_numpy(stacked[i:i + 256])) for i in range(0, len(stacked), 256)])
        assert torch.equal(vs.file_outputs(f), want), f"file {f}"


def _run_equals_the_pipeline(cfg, files, vs, trials):
    runs = vs.run(trials)
    taus = [t.get("tau_active", None) for t in trials]
    lines = 0
    default_tau = cfg.tau_active
    try:
        for f, (uri, x, _) in enumerate(files):
            fw = file_windows(x, cfg)
            for t, tau in enumerate(taus):
                want = pipeline_prediction(cfg, fw, uri, default_tau if tau is None else tau)
                got = runs[f][t]
                assert got.to_rttm() == want.to_rttm(), f"file {f} trial {t}"
                assert (got.uri, got.modality) == (want.uri, want.modality) == (uri, "speech"), f"file {f} trial {t}"
                lines += got.to_rttm().count("\n")
    finally:
        cfg.tau_active = default_tau
    return runs, lines


def test_run_equals_the_pipeline(dataset):
    cfg, files, vs, trials = dataset
    runs, lines = _run_equals_the_pipeline(cfg, files, vs, trials)
    assert lines > 100
    assert all(r[2].to_rttm() == "" for r in runs), "tau_active = 1: no speech"


@pytest.mark.parametrize("latency", [2.0, "max"])
def test_run_equals_the_pipeline_at_other_latencies(latency, oracle_nets, cuda_device):
    cfg = make_config(oracle_nets, cuda_device, latency=latency)
    files = [make_files()[i] for i in (0, 2, 3)]
    vs = VoiceActivitySweep(cfg, files)
    _, lines = _run_equals_the_pipeline(cfg, files, vs, as_trials([None, 0.0, 0.35, 0.6, 0.8]))
    assert lines > 20


def test_chunk_turns_equal_the_device_post_path(dataset):
    cfg, files, vs, trials = dataset
    taus = np.array([t.get("tau_active", cfg.tau_active) for t in trials])
    r = vs.binarize(taus)
    lib = _lib.lib()
    F = vs.seg.shape[1]
    nw = int(round(cfg.latency / cfg.step))
    for f in (0, 2, 3):
        c0, c1 = int(vs.offsets[f]), int(vs.offsets[f + 1])
        fw = file_windows(files[f][1], cfg)
        vad = vs.file_outputs(f).amax(dim=-1, keepdim=True).contiguous()
        maps = torch.zeros((c1 - c0, 1), dtype=torch.int32, device=vad.device)
        for t, tau in enumerate(taus):
            post = DevicePostPath(cfg.step, cfg.latency, tau, F, 1, 1, vad.device)
            assert post.nw == nw
            for b0 in range(0, c1 - c0, 256):
                B = min(256, c1 - c0 - b0)
                starts = fw.starts[b0:b0 + B]
                plan, _, _ = post.plan(starts, seg_resolution(cfg, float(starts[0]), F))
                assert np.array_equal(plan, vs.plan[c0 + b0:c0 + b0 + B])
                header, turns = post.buffers(B)
                n = ctypes.c_int()
                with torch.cuda.device(vad.device):
                    _lib.check(lib.dg_post_step(post.handle, vad[b0:].data_ptr(), maps[b0:].data_ptr(), B, plan.ctypes.data,
                                                header.ctypes.data, turns.ctypes.data, len(turns), ctypes.byref(n),
                                                _lib.stream_ptr(vad.device)))
                for c in range(B):
                    o, k, frames, _ = header[c].tolist()
                    go, gk, gframes, zero = r.header[t, c0 + b0 + c].tolist()
                    assert (gk, gframes, zero) == (k, frames, 0), (f, t, c)
                    assert r.turns[go:go + gk].tolist() == turns[o:o + k].tolist(), (f, t, c)


def test_components_equal_the_oracle(dataset):
    cfg, files, vs, trials = dataset
    per_file, total = vs.score(trials)
    runs = vs.run(trials)
    assert set(vs.timing) >= {"network", "curve", "score", "sweep"}
    fold = per_file[0].as_array()
    for f, (_, _, ref) in enumerate(files):
        want = np.stack([detection_components(ref, p) for p in runs[f]])
        got = per_file[f].as_array()
        assert np.array_equal(got, want), (f, np.argwhere(got != want))
        assert got[2, 0] == 0.0 and got[2, 1] == got[2, 2] > 0, "tau_active = 1: all missed"
        if f:
            fold = fold + got
    assert np.array_equal(total.as_array(), fold)
    assert len(set(total.detection_error_rate.tolist())) >= 6


def test_one_trial_among_300_one_file_alone_and_file_order(dataset, oracle_nets, cuda_device):
    cfg, files, vs, trials = dataset
    rng = np.random.default_rng(23)
    many = as_trials(rng.uniform(0.0, 1.0, 300).tolist())
    many[:len(trials)] = trials
    big, _ = vs.score(many)
    for t in (0, 2, 8, 9, 137, 299):
        small, _ = vs.score(many[t:t + 1])
        for f in range(len(files)):
            assert np.array_equal(small[f].as_array()[0], big[f].as_array()[t]), (f, t)
    want_run = [[p.to_rttm() for p in r] for r in vs.run(trials)]
    one = VoiceActivitySweep(cfg, [files[3]])
    per_file, total = one.score(trials)
    assert np.array_equal(per_file[0].as_array(), big[3].as_array()[:len(trials)])
    assert np.array_equal(total.as_array(), per_file[0].as_array())
    assert [p.to_rttm() for p in one.run(trials)[0]] == want_run[3]
    rev = VoiceActivitySweep(cfg, files[::-1])
    per_file, _ = rev.score(trials)
    n = len(files)
    for f in range(n):
        assert np.array_equal(per_file[n - 1 - f].as_array(), big[f].as_array()[:len(trials)]), f"file {f}"
    assert [[p.to_rttm() for p in r] for r in rev.run(trials)[::-1]] == want_run


def test_scoring_runs_no_network_work(dataset):
    cfg, files, vs, trials = dataset
    lib = _lib.lib()
    small = VoiceActivitySweep(cfg, files[:3])
    deltas = []
    for d in (small, vs):
        d.score(trials[:4])                                   # first use: buffers sized
        before = lib.dg_launch_count()
        d.score(trials[:4])
        deltas.append(lib.dg_launch_count() - before)
    assert deltas[0] == deltas[1] > 0
    a, _ = vs.score(trials)
    b, _ = vs.score(trials)
    assert all(np.array_equal(x.as_array(), y.as_array()) for x, y in zip(a, b))


def test_files_without_a_reference_run_but_do_not_score(dataset):
    cfg, files, vs, trials = dataset
    part = VoiceActivitySweep(cfg, [(files[0][0], files[0][1], None), files[4]])
    with pytest.raises(ValueError, match="without a reference"):
        part.score(trials)
    want = [[p.to_rttm() for p in r] for r in vs.run(trials[:3])]
    runs = part.run(trials[:3])
    assert [p.to_rttm() for p in runs[0]] == want[0] and [p.to_rttm() for p in runs[1]] == want[4]


def test_argument_checks_never_launch(dataset):
    cfg, files, vs, _ = dataset
    lib = _lib.lib()
    N, F, K = vs.seg.shape
    nf = len(files)
    h = vs._h
    header = np.zeros((1, N, 4), np.int32)
    turns = np.zeros(1 << 20, np.uint32)
    comp = np.zeros((nf, 2, 2))
    n = ctypes.c_int()
    rows = np.array([[0.0, 1.0], [2.0, 3.0]] * nf)
    good_roff = np.arange(0, 2 * nf + 1, 2, dtype=np.int32)

    def c(a, dtype):
        return np.ascontiguousarray(a, dtype=dtype)

    def curve(off=vs.offsets, plan=vs.plan, n_chunks=N, handle=h):
        off, plan = c(off, np.int32), c(plan, np.int32)
        return lib.dg_vad_sweep_curve(handle, vs.seg.data_ptr(), n_chunks, len(off) - 1, off.ctypes.data, plan.ctypes.data,
                                      None)

    def run(taus=np.array([0.5]), T=1):
        taus = c(taus, np.float64)
        return lib.dg_vad_sweep_run_files(h, taus.ctypes.data, T, header.ctypes.data, turns.ctypes.data, len(turns),
                                          ctypes.byref(n), None)

    def score(taus=np.array([0.5]), T=1, shifts=vs.shifts, start=vs.out_start, roff=good_roff, r=rows, collar=PATCH_COLLAR):
        taus, shifts, start, roff, r = (c(taus, np.float64), c(shifts, np.float64), c(start, np.float64), c(roff, np.int32),
                                        c(r, np.float64))
        return lib.dg_vad_sweep_score_files(h, taus.ctypes.data, T, start.ctypes.data, vs.out_res.ctypes.data,
                                            shifts.ctypes.data, collar, r.ctypes.data, roff.ctypes.data, comp.ctypes.data,
                                            None)

    assert run() == 0 and score() == 0
    dup = vs.offsets.copy()
    dup[2] = dup[1]
    reach = vs.plan.copy()
    reach[int(vs.offsets[2]), 0] = 2                          # a file's first chunk aggregating the previous file's last
    wide = vs.plan.copy()
    wide[5, 1] = 1024
    bad_shift = vs.shifts.copy()
    bad_shift[1] = np.nan
    bad_time = vs.out_start.copy()
    bad_time[7] = np.inf
    overlap = rows.copy()
    overlap[7] = [0.5, 3.0]                                   # file 3: rows that overlap
    close = rows.copy()
    close[5] = [1.0 + 5e-7, 3.0]                              # file 2: a gap of 5e-7 s, not a support
    reversed_row = rows.copy()
    reversed_row[0] = [1.0, 0.0]
    shrinking = good_roff.copy()
    shrinking[2] = 1
    cases = [(curve, "dg_vad_sweep_curve", kw, name) for name, kw in {
        "file without chunks": dict(off=dup), "offsets not ending at N": dict(off=np.append(vs.offsets[:-1], N - 1)),
        "N = 0": dict(n_chunks=0, off=np.zeros(nf + 1)), "plan reaches into the previous file": dict(plan=reach),
        "more than 1023 frames": dict(plan=wide), "no handle": dict(handle=None),
    }.items()] + [(run, "dg_vad_sweep_run_files", kw, name) for name, kw in {
        "T = 0": dict(T=0), "T > 65535": dict(T=65536), "tau not finite": dict(taus=np.array([np.nan])),
    }.items()] + [(score, "dg_vad_sweep_score_files", kw, name) for name, kw in {
        "T = 0": dict(T=0), "tau not finite": dict(taus=np.array([np.inf])), "shift not finite": dict(shifts=bad_shift),
        "chunk time not finite": dict(start=bad_time), "collar < 0": dict(collar=-0.1),
        "rows overlap": dict(r=overlap), "rows closer than 1e-6 s": dict(r=close), "row reversed": dict(r=reversed_row),
        "reference offsets decrease": dict(roff=shrinking), "reference offsets not starting at 0": dict(roff=good_roff + 1),
    }.items()]
    for fn, who, kw, name in cases:
        before = lib.dg_launch_count()
        rc = fn(**kw)
        assert rc == -1 and lib.dg_launch_count() == before, name
        assert who.encode() in lib.dg_last_error(), name
    assert run() == 0 and curve() == 0                       # the handle still works after every refusal
