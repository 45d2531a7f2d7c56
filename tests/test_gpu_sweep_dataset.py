"""Dataset sweep on the device (dg_sweep_run_files / dg_sweep_score_files through diart_b200.tune.DatasetSweep): for every
file and trial the resident network outputs, maps, centroids, predictions and DER components are the bits a
HyperParameterSweep of that file alone gives, whatever the other files, their order and the number of trials; scoring runs
no network kernel; bad arguments never launch."""
import ctypes

import numpy as np
import pytest
import torch

from diart_b200 import _lib, synth
from diart_b200.tune import PATCH_COLLAR, DatasetSweep, HyperParameterSweep, file_windows, trial_params
from oracle.clustering import OracleClustering
from test_gpu_sweep import TRIALS, make_config
from test_gpu_sweep_score import oracle_rows, synth_reference

pytestmark = pytest.mark.gpu

# seconds: one window with left padding; exactly 256 windows; 257 windows (a second network batch of one); 601 windows with
# an incomplete last block; two others
SECONDS = (3.2, 132.3, 132.8, 304.7, 61.3, 47.9)


def make_files():
    files = []
    for i, secs in enumerate(SECONDS):
        x = synth.synth_audio(int(secs * 16000), seed=900 + i, num_speakers=3 + i % 3)
        files.append((f"file{i}", x, synth_reference(60 + i, 3 + i % 4, secs, uri=f"file{i}")))
    return files


@pytest.fixture(scope="module")
def dataset(oracle_nets, cuda_device):
    cfg = make_config(oracle_nets, cuda_device)
    files = make_files()
    ds = DatasetSweep(cfg, files)
    alone = HyperParameterSweep(cfg)
    want_score = [alone.score(x, ref, TRIALS).as_array() for _, x, ref in files]
    want_run = [[p.to_rttm() for p in alone.run(x, uri=uri, trials=TRIALS)] for uri, x, _ in files]
    return cfg, files, ds, alone, want_score, want_run


def test_windows_of_the_chosen_lengths(oracle_nets, cuda_device):
    cfg = make_config(oracle_nets, cuda_device)
    fws = [file_windows(np.zeros(int(s * 16000), np.float32), cfg) for s in SECONDS]
    assert [fw.num_windows for fw in fws[:4]] == [1, 256, 257, 601]
    assert fws[0].padding[0] > 0 and all(fw.padding[0] == 0 for fw in fws[1:])


def test_resident_outputs_equal_the_per_file_network_pass(dataset):
    cfg, files, ds, alone, _, _ = dataset
    assert ds.num_chunks == sum(file_windows(x, cfg).num_windows for _, x, _ in files)
    N, F, K = ds.seg.shape
    assert ds.resident_bytes == N * (F * K + K * ds.emb.shape[2]) * 4
    for f, (_, x, _) in enumerate(files):
        seg, emb = alone.network_pass(file_windows(x, cfg))
        got_seg, got_emb = ds.file_outputs(f)
        assert torch.equal(got_seg, seg) and torch.equal(got_emb, emb), f"file {f}"


def test_components_and_predictions_equal_each_file_alone(dataset):
    cfg, files, ds, alone, want_score, want_run = dataset
    per_file, total = ds.score(TRIALS)
    assert len(per_file) == len(files)
    fold = per_file[0].as_array()
    for f, (uri, x, ref) in enumerate(files):
        assert np.array_equal(per_file[f].as_array(), want_score[f]), f"file {f}"
        if f:
            fold = fold + per_file[f].as_array()
    assert np.array_equal(total.as_array(), fold)
    runs = ds.run(TRIALS)
    assert [[p.to_rttm() for p in r] for r in runs] == want_run
    for f, (uri, x, ref) in enumerate(files):           # and the host oracle on those predictions
        assert np.array_equal(per_file[f].as_array(), oracle_rows(ref, runs[f])), f"file {f}"
    assert sum(r.count("\n") for rr in want_run for r in rr) > 200


def test_score_files_equals_the_dataset_sweep(dataset):
    cfg, files, ds, alone, want_score, _ = dataset
    per_file, total = alone.score_files([(x, ref) for _, x, ref in files[:3]], TRIALS)
    assert all(np.array_equal(per_file[f].as_array(), want_score[f]) for f in range(3))
    assert np.array_equal(total.as_array(), want_score[0] + want_score[1] + want_score[2])
    assert set(alone.timing) == {"network", "score"}


def test_clustering_equals_the_oracle(dataset):
    cfg, files, ds, alone, _, _ = dataset
    params = trial_params(TRIALS, cfg)
    r = ds.sweep(params, keep_state=True)
    maps, centers = r.maps.cpu().numpy(), r.centers.cpu().numpy()
    assert centers.shape[:2] == (len(files), len(params))
    for f in range(len(files)):
        c0, c1 = int(ds.offsets[f]), int(ds.offsets[f + 1])
        s_np, e_np = (t.cpu().numpy() for t in ds.file_outputs(f))
        for t, (tau, rho, delta) in enumerate(params):
            replay = OracleClustering(tau, rho, delta, "cosine", cfg.max_speakers)
            want = np.stack([replay(s, e)[0] for s, e in zip(s_np, e_np)])
            assert np.array_equal(maps[t, c0:c1], want), f"file {f} trial {t}: maps"
            assert np.array_equal(centers[f, t], replay.centers), f"file {f} trial {t}: centroids"


def test_one_file_alone_and_file_order(dataset, oracle_nets, cuda_device):
    cfg, files, ds, alone, want_score, want_run = dataset
    one = DatasetSweep(cfg, [files[3]])
    per_file, total = one.score(TRIALS)
    assert np.array_equal(per_file[0].as_array(), want_score[3]) and np.array_equal(total.as_array(), want_score[3])
    assert [p.to_rttm() for p in one.run(TRIALS)[0]] == want_run[3]
    rev = DatasetSweep(cfg, files[::-1])
    per_file, total = rev.score(TRIALS)
    n = len(files)
    for f in range(n):
        assert np.array_equal(per_file[n - 1 - f].as_array(), want_score[f]), f"file {f}"
    runs = rev.run(TRIALS[:3])
    assert [[p.to_rttm() for p in r] for r in runs[::-1]] == [w[:3] for w in want_run]


def test_one_trial_alone_equals_the_same_trial_among_300(dataset):
    """300 trials x 6 files = 1800 states: several waves of the clustering launch"""
    cfg, files, ds, alone, _, _ = dataset
    rng = np.random.default_rng(17)
    many = np.column_stack([rng.uniform(0.3, 0.8, 300), rng.uniform(0, 1, 300), rng.uniform(0.05, 2, 300)])
    many[:len(TRIALS)] = trial_params(TRIALS, cfg)
    as_trials = [dict(zip(("tau_active", "rho_update", "delta_new"), p)) for p in many.tolist()]
    big, _ = ds.score(as_trials)
    big_run = ds.sweep(many, keep_state=True)
    for t in (0, 4, 6, 137, 299):
        small, _ = ds.score(as_trials[t:t + 1])
        for f in range(len(files)):
            assert np.array_equal(small[f].as_array()[0], big[f].as_array()[t]), (f, t)
        one = ds.sweep(many[t:t + 1], keep_state=True)
        assert torch.equal(one.maps[0], big_run.maps[t]) and torch.equal(one.centers[:, 0], big_run.centers[:, t]), t


def test_repeated_scoring_runs_no_network_work(dataset):
    cfg, files, ds, alone, _, _ = dataset
    lib = _lib.lib()
    small = DatasetSweep(cfg, files[:3])
    deltas = []
    for d in (small, ds):
        d.score(TRIALS[:4])                                   # first use: buffers sized
        before = lib.dg_launch_count()
        d.score(TRIALS[:4])
        deltas.append(lib.dg_launch_count() - before)
    assert deltas[0] == deltas[1] > 0
    a, _ = ds.score(TRIALS)
    b, _ = ds.score(TRIALS)
    assert all(np.array_equal(x.as_array(), y.as_array()) for x, y in zip(a, b))


@pytest.mark.parametrize("kw", [{"latency": 2.0}, {"max_speakers": 4}])
def test_other_configurations_against_a_seven_label_reference(kw, oracle_nets, cuda_device):
    cfg = make_config(oracle_nets, cuda_device, **kw)
    files = [(uri, x, synth_reference(70 + i, 7, len(x) / 16000, uri=uri)) for i, (uri, x, _) in
             enumerate(make_files()[:3])]
    ds = DatasetSweep(cfg, files)
    trials = TRIALS[:6]
    per_file, total = ds.score(trials)
    runs = ds.run(trials)
    alone = HyperParameterSweep(cfg)
    for f, (uri, x, ref) in enumerate(files):
        assert np.array_equal(per_file[f].as_array(), alone.score(x, ref, trials).as_array()), f"file {f}"
        assert [p.to_rttm() for p in runs[f]] == [p.to_rttm() for p in alone.run(x, uri=uri, trials=trials)], f"file {f}"


def test_files_without_a_reference_run_but_do_not_score(dataset, oracle_nets, cuda_device):
    cfg, files, ds, alone, _, want_run = dataset
    part = DatasetSweep(cfg, [(files[0][0], files[0][1], None), files[4]])
    with pytest.raises(ValueError, match="without a reference"):
        part.score(TRIALS)
    runs = part.run(TRIALS[:2])
    assert [p.to_rttm() for p in runs[0]] == want_run[0][:2] and [p.to_rttm() for p in runs[1]] == want_run[4][:2]


def test_argument_checks_never_launch(dataset):
    cfg, files, ds, alone, _, _ = dataset
    lib = _lib.lib()
    N, F, K = ds.seg.shape
    nf = len(files)
    h, _ = alone._handle(F, K, ds.emb.shape[2])
    header = np.zeros((1, N, 4), np.int32)
    turns = np.zeros(1 << 20, np.uint32)
    comp = np.zeros((nf, 2, 5))
    n = ctypes.c_int()
    rows = np.array([[0.0, 1.0], [2.0, 3.0]] * nf)
    good_labels = np.zeros(2 * nf, np.int32)
    good_roff = np.arange(0, 2 * nf + 1, 2, dtype=np.int32)
    good_counts = np.ones(nf, np.int32)

    def c(a, dtype):
        return np.ascontiguousarray(a, dtype=dtype)

    def run(off=ds.offsets, T=1, n_chunks=N, params=np.array([[0.5, 0.3, 1.0]])):
        off, params = c(off, np.int32), c(params, np.float64)
        return lib.dg_sweep_run_files(h, ds.seg.data_ptr(), ds.emb.data_ptr(), n_chunks, len(off) - 1, off.ctypes.data,
                                      params.ctypes.data, T, ds.plan.ctypes.data, None, None, header.ctypes.data,
                                      turns.ctypes.data, len(turns), ctypes.byref(n), None)

    def score(off=ds.offsets, T=1, shifts=ds.shifts, labels=good_labels, roff=good_roff, counts=good_counts, r=rows,
              params=np.array([[0.5, 0.3, 1.0]])):
        off, params, shifts = c(off, np.int32), c(params, np.float64), c(shifts, np.float64)
        labels, roff, counts, r = c(labels, np.int32), c(roff, np.int32), c(counts, np.int32), c(r, np.float64)
        return lib.dg_sweep_score_files(h, ds.seg.data_ptr(), ds.emb.data_ptr(), N, len(off) - 1, off.ctypes.data,
                                        params.ctypes.data, T, ds.plan.ctypes.data, ds.out_start.ctypes.data,
                                        ds.out_res.ctypes.data, shifts.ctypes.data, PATCH_COLLAR, r.ctypes.data,
                                        labels.ctypes.data, roff.ctypes.data, counts.ctypes.data, comp.ctypes.data, None,
                                        None, 0, None)

    assert run() == 0 and score() == 0
    dup = ds.offsets.copy()
    dup[2] = dup[1]
    back = ds.offsets.copy()
    back[2], back[3] = back[3], back[2]
    bad_shift = ds.shifts.copy()
    bad_shift[1] = np.nan
    wide = good_counts.copy()
    wide[2] = 33
    outside = good_labels.copy()
    outside[5] = 1                                            # file 2's row 1 with one label only
    overlap = rows.copy()
    overlap[7] = [0.5, 3.0]                                   # file 3: two rows of label 0 that overlap
    shrinking = good_roff.copy()
    shrinking[2] = 1
    assert 33 * 65535 > (1 << 21)
    common = {
        "file without chunks": dict(off=dup), "offsets not increasing": dict(off=back),
        "offsets not ending at N": dict(off=np.append(ds.offsets[:-1], N - 1)),
        "offsets not starting at 0": dict(off=np.append([1], ds.offsets[1:])),
        "too many states": dict(off=np.append(np.arange(33), N), T=65535, params=np.tile([[0.5, 0.3, 1.0]], (65535, 1))),
        "T = 0": dict(T=0), "param not finite": dict(params=np.array([[0.5, np.inf, 1.0]])),
    }
    cases = [(run, "dg_sweep_run_files", kw, name) for name, kw in common.items()] + \
            [(run, "dg_sweep_run_files", dict(n_chunks=0), "N = 0")] + \
            [(score, "dg_sweep_score_files", kw, name) for name, kw in common.items()] + \
            [(score, "dg_sweep_score_files", kw, name) for name, kw in {
                "shift not finite": dict(shifts=bad_shift), "more than 32 labels": dict(counts=wide),
                "label outside its file's range": dict(labels=outside), "rows of a label overlap": dict(r=overlap),
                "reference offsets decrease": dict(roff=shrinking),
                "reference offsets not starting at 0": dict(roff=good_roff + 1, r=np.vstack([rows, [[8.0, 9.0]]]),
                                                            labels=np.append(good_labels, 0)),
            }.items()]
    for fn, who, kw, name in cases:
        before = lib.dg_launch_count()
        rc = fn(**kw)
        assert rc == -1 and lib.dg_launch_count() == before, name
        assert who.encode() in lib.dg_last_error(), name
