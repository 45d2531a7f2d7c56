"""Hyper-parameter sweep on the device (dg_sweep_run through diart_b200.tune.HyperParameterSweep): every trial's whole-file
prediction equals a SpeakerDiarization run with that trial's parameters; clustering equals the oracle bit for bit; the
post-path equals the reference-pinned host blocks; launch geometry does not change results."""
import ctypes

import numpy as np
import pytest
import torch

from diart_b200 import _lib, blocks, models, synth
from diart_b200.blocks.post import post_plan, turn_times
from diart_b200.core import SlidingWindow, SlidingWindowFeature
from diart_b200.sinks import PredictionAccumulator
from diart_b200.tune import HyperParameterSweep, assemble_predictions, file_windows, trial_params
from oracle.clustering import OracleClustering

pytestmark = pytest.mark.gpu

TRIALS = [
    {},                                                     # the config's values
    {"tau_active": 0.45, "rho_update": 0.1, "delta_new": 0.6},
    {"tau_active": 0.7, "rho_update": 0.5, "delta_new": 1.4},
    {"tau_active": 0.55, "rho_update": 0.2, "delta_new": 1.9},
    {"tau_active": 0.6, "rho_update": 0.3, "delta_new": 1e-3},   # every active speaker is new until the table is full
    {"tau_active": 0.5, "rho_update": 1.0, "delta_new": 0.8},    # no centroid is ever updated
    {"tau_active": 1.0},                                         # no speaker is active
    {"tau_active": 0.35, "rho_update": 0.05, "delta_new": 1.0},
    {"rho_update": 0.0, "delta_new": 2.0},
]


def make_config(oracle_nets, device, **kw):
    seg_o, emb_o = oracle_nets
    return blocks.SpeakerDiarizationConfig(
        segmentation=models.SegmentationModel(models.B200SegmentationLoader(seg_o.state_dict())),
        embedding=models.EmbeddingModel(models.B200EmbeddingLoader(emb_o.state_dict())), device=device, **kw)


def pipeline_prediction(config, fw, uri):
    """Benchmark.run_single with SpeakerDiarization(config) over the sweep's windows, batches of 256"""
    pipe = blocks.SpeakerDiarization(config)
    pipe.set_timestamp_shift(-fw.padding[0])
    acc = PredictionAccumulator(uri)
    sr = config.sample_rate
    chunks = [SlidingWindowFeature(fw.window(i)[:, None], SlidingWindow(start=fw.starts[i], duration=1 / sr, step=1 / sr))
              for i in range(fw.num_windows)]
    for i in range(0, len(chunks), 256):
        for out in pipe(chunks[i:i + 256]):
            acc.on_next(out)
    return acc.get_prediction()


def chunk_turns(r, t, N):
    """trial t's turns per chunk as sorted (speaker, on time, off time) lists"""
    rows, g, a, b = turn_times(r.header.reshape(-1, 4), r.turns, r.n_turns, r.out_start, r.out_res)
    sel = rows // N == t
    out = [[] for _ in range(N)]
    for c, k, x, y in zip((rows[sel] % N).tolist(), g[sel].tolist(), a[sel].tolist(), b[sel].tolist()):
        out[c].append((k, x, y))
    return [sorted(o) for o in out]


@pytest.fixture(scope="module")
def file_600(oracle_nets, cuda_device):
    """a 304.7 s file (601 chunks at the default config, the last block incomplete), 5 speakers, through the sweep's network pass"""
    x = synth.synth_audio(int(304.7 * 16000), seed=4242, num_speakers=5)
    cfg = make_config(oracle_nets, cuda_device)
    sweep = HyperParameterSweep(cfg)
    fw = file_windows(x, cfg)
    assert fw.num_windows >= 600
    seg, emb = sweep.network_pass(fw)
    return x, cfg, sweep, fw, seg, emb


def test_whole_file_predictions_equal_the_pipeline(file_600, oracle_nets, cuda_device):
    x, cfg, sweep, fw, seg, emb = file_600
    got = sweep.run(x, uri="synth", trials=TRIALS)
    params = trial_params(TRIALS, cfg)
    lines = 0
    for t, p in enumerate(params):
        c = make_config(oracle_nets, cuda_device, tau_active=p[0], rho_update=p[1], delta_new=p[2])
        want = pipeline_prediction(c, fw, "synth").to_rttm()
        assert got[t].to_rttm() == want, f"trial {t} {TRIALS[t]}"
        lines += want.count("\n")
    if float(seg.max()) < 1.0:
        assert got[6].to_rttm() == ""
    assert lines > 100
    print(f"sweep timing {sweep.timing}, {lines} RTTM lines over {len(TRIALS)} trials")


def test_clustering_equals_the_oracle(file_600):
    x, cfg, sweep, fw, seg, emb = file_600
    params = trial_params(TRIALS, cfg)
    r = sweep.sweep(seg, emb, fw.starts, params, keep_state=True)
    s_np, e_np = seg.cpu().numpy(), emb.cpu().numpy()
    maps, centers = r.maps.cpu().numpy(), r.centers.cpu().numpy()
    for t, (tau, rho, delta) in enumerate(params):
        replay = OracleClustering(tau, rho, delta, "cosine", cfg.max_speakers)
        want = np.stack([replay(s, e)[0] for s, e in zip(s_np, e_np)])
        assert np.array_equal(maps[t], want), f"trial {t}: maps"
        assert np.array_equal(centers[t], replay.centers), f"trial {t}: centroids"
    assert len({maps[t].tobytes() for t in range(len(params))}) >= 5, "the trials must lead to different clusterings"


def test_post_path_equals_the_host_blocks_on_oracle_maps(file_600):
    x, cfg, sweep, fw, seg, emb = file_600
    params = trial_params(TRIALS[1:3], cfg)
    r = sweep.sweep(seg, emb, fw.starts, params)
    s_np, e_np = seg.cpu().numpy(), emb.cpu().numpy()
    N, F = s_np.shape[:2]
    res = 5.0 / F
    for t, (tau, rho, delta) in enumerate(params):
        replay = OracleClustering(tau, rho, delta, "cosine", cfg.max_speakers)
        agg = blocks.DelayedAggregation(cfg.step, cfg.latency, strategy="hamming", cropping_mode="loose")
        binarize = blocks.Binarize(tau)
        got, buf, n = chunk_turns(r, t, N), [], 0
        for i in range(N):
            permuted = np.zeros((F, cfg.max_speakers))
            for k, g in enumerate(replay(s_np[i], e_np[i])[0]):
                if g >= 0:
                    permuted[:, g] = s_np[i][:, k]
            buf.append(SlidingWindowFeature(permuted, SlidingWindow(start=fw.starts[i], duration=res, step=res)))
            want = sorted((int(lab[7:]), s.start, s.end) for s, _, lab in binarize(agg(buf)).itertracks(yield_label=True))
            assert got[i] == want, f"trial {t} chunk {i}"
            n += len(want)
            if len(buf) == agg.num_overlapping_windows:
                buf = buf[1:]
        assert n > N // 2


def test_launch_geometry_does_not_change_results(file_600):
    """a trial alone (T = 1) and inside T = 300 (more trials than resident CTAs: several waves) give the same bits"""
    x, cfg, sweep, fw, seg, emb = file_600
    rng = np.random.default_rng(5)
    many = np.column_stack([rng.uniform(0.3, 0.8, 300), rng.uniform(0, 1, 300), rng.uniform(0.05, 2, 300)])
    many[:len(TRIALS)] = trial_params(TRIALS, cfg)
    big = sweep.sweep(seg, emb, fw.starts, many, keep_state=True)
    N = seg.shape[0]
    labels = [f"speaker{g}" for g in range(cfg.max_speakers)]
    rttm_big = assemble_predictions(big.header, big.turns, big.n_turns, big.out_start, big.out_res, labels)
    for t in (0, 4, 5, 6, 137, 299):
        one = sweep.sweep(seg, emb, fw.starts, many[t:t + 1], keep_state=True)
        assert torch.equal(one.maps[0], big.maps[t]) and torch.equal(one.centers[0], big.centers[t]), f"trial {t}"
        assert chunk_turns(one, 0, N) == chunk_turns(big, t, N), f"trial {t}"
        got = assemble_predictions(one.header, one.turns, one.n_turns, one.out_start, one.out_res, labels)[0]
        assert got.to_rttm() == rttm_big[t].to_rttm()


@pytest.mark.parametrize("kw", [{"latency": 2.0}, {"max_speakers": 4}])
def test_other_configurations_equal_the_pipeline(kw, oracle_nets, cuda_device):
    x = synth.synth_audio(int(152.3 * 16000), seed=99, num_speakers=6)
    cfg = make_config(oracle_nets, cuda_device, **kw)
    sweep = HyperParameterSweep(cfg)
    fw = file_windows(x, cfg)
    trials = [{}, {"tau_active": 0.45, "rho_update": 0.1, "delta_new": 0.5}, {"delta_new": 1e-3},
              {"tau_active": 0.7, "rho_update": 1.0, "delta_new": 1.5}]
    got = sweep.run(x, uri="f", trials=trials)
    for t, p in enumerate(trial_params(trials, cfg)):
        c = make_config(oracle_nets, cuda_device, tau_active=p[0], rho_update=p[1], delta_new=p[2], **kw)
        assert got[t].to_rttm() == pipeline_prediction(c, fw, "f").to_rttm(), f"trial {t} {trials[t]}"


def test_many_turns_need_a_second_copy_in_the_sweep(file_600):
    """more turns than the prefix that travels with the headers, and more than the host buffer first offered"""
    x, cfg, sweep, fw, seg, emb = file_600
    params = np.tile([[0.3, 0.3, 1.0]], (64, 1))
    sweep._turns = np.empty(16, dtype=np.uint32)
    r = sweep.sweep(seg, emb, fw.starts, params)
    assert r.n_turns > 16384
    first = chunk_turns(r, 0, seg.shape[0])
    assert all(chunk_turns(r, t, seg.shape[0]) == first for t in (31, 63)), "identical trials must give identical turns"


def test_run_time_argument_checks_never_launch(file_600):
    x, cfg, sweep, fw, seg, emb = file_600
    lib = _lib.lib()
    N, F, K = seg.shape
    h, nw = sweep._handle(F, K, emb.shape[2])
    plan = np.zeros((N, 4 + nw), np.int32)
    header = np.zeros((4, N, 4), np.int32)
    turns = np.zeros(1024, np.uint32)
    n = ctypes.c_int()
    good = np.array([[0.5, 0.3, 1.0]])
    cases = [(good, 0, N), (good, 1, 0), (np.array([[np.nan, 0.3, 1.0]]), 1, N), (np.array([[0.5, np.inf, 1.0]]), 1, N),
             (np.array([[0.5, 0.3, -np.inf]]), 1, N)]
    for params, T, n_chunks in cases:
        before = lib.dg_launch_count()
        rc = lib.dg_sweep_run(h, seg.data_ptr(), emb.data_ptr(), n_chunks, params.ctypes.data, T, plan.ctypes.data, None,
                              None, header.ctypes.data, turns.ctypes.data, len(turns), ctypes.byref(n), None)
        assert rc == -1 and lib.dg_launch_count() == before, (params, T, n_chunks)
        assert b"dg_sweep_run" in lib.dg_last_error()
    # plan rows the file's chunks cannot have: more buffers than latency / step, buffers before the file's first chunk, F + 2
    # output frames, and (two files) the second file's first chunk reaching into the first file; at latency = 4 steps
    h, nw = sweep._handle(F, K, emb.shape[2], 4)
    plan = np.ascontiguousarray(post_plan(fw.starts, sweep._seg_resolution(float(fw.starts[0]), F), np.zeros(0), np.zeros(0),
                                          nw, F, cfg.step, nw * cfg.step)[0])
    wide, early, long_first = plan.copy(), plan.copy(), plan.copy()
    wide[N - 1, 0] = nw + 1
    early[1, 0] = 3
    long_first[0, 2] = F + 2
    two_files = np.array([0, 300, N], np.int32)
    for name, bad, offs in (("nb > nw", wide, None), ("before the first chunk", early, None), ("F + 2 frames", long_first, None),
                            ("into the previous file", plan, two_files)):
        before = lib.dg_launch_count()
        if offs is None:
            rc = lib.dg_sweep_run(h, seg.data_ptr(), emb.data_ptr(), N, good.ctypes.data, 1, bad.ctypes.data, None, None,
                                  header.ctypes.data, turns.ctypes.data, len(turns), ctypes.byref(n), None)
        else:
            rc = lib.dg_sweep_run_files(h, seg.data_ptr(), emb.data_ptr(), N, len(offs) - 1, offs.ctypes.data, good.ctypes.data,
                                        1, bad.ctypes.data, None, None, header.ctypes.data, turns.ctypes.data, len(turns),
                                        ctypes.byref(n), None)
        assert rc == -1 and lib.dg_launch_count() == before, name
        assert b": plan row" in lib.dg_last_error(), name
