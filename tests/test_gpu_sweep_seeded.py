"""Seeded dataset sweeps and the identification error rate on the device (DatasetSweep(speakers=...), dg_sweep_set_seeds,
dg_sweep_set_identities): every (file, trial) clustering starts from its file's known centroids exactly as a pipeline with
set_known_speakers does -- predictions, maps and centroids bit for bit -- files without seeds keep the unseeded bits, the
identification error components equal the protocol oracle's, and bad arguments never launch."""
import ctypes
import itertools

import numpy as np
import pytest

from diart_b200 import _lib, blocks
from diart_b200.core import Annotation, SlidingWindow, SlidingWindowFeature
from diart_b200.sinks import PredictionAccumulator
from diart_b200.speakers import KnownSpeakers, speaker_labels
from diart_b200.tune import (DatasetSweep, DiarizationErrorRate, HyperParameterSweep, IdentificationErrorComponents,
                             IdentificationErrorRate, file_windows, trial_params)
from ier_oracle import protocol_ier_components
from test_gpu_known_speakers import seeded_oracle
from test_gpu_sweep import TRIALS, make_config
from test_gpu_sweep_dataset import SECONDS, make_files
from test_gpu_sweep_protocol import UEMS
from test_gpu_sweep_score import synth_reference
from test_sweep_seeded_host import der_mapping

pytestmark = pytest.mark.gpu

NAMES = [["alice", "bob"], None, ["alice", "bob", "carol"], ["dave", "erin", "frank", "grace"], [], ["carol", "dave"]]
ROWS = [[0, 1], None, [0, 1, 2], [1, 2, 3, 0], [], [2, 3]]      # which learned centroids each file's names take
PRED_TRIALS = [0, 4, 5]     # the config, delta_new = 1e-3 (every speaker new until full), rho_update = 1 (no update)


def known_speakers(pool):
    out = []
    for names, rows in zip(NAMES, ROWS):
        if names is None:
            out.append(None)
        elif not names:
            out.append(KnownSpeakers([], np.zeros((0, 0))))
        else:
            out.append(KnownSpeakers(names, pool[rows]))
    return out


@pytest.fixture(scope="module")
def seeded(oracle_nets, cuda_device):
    cfg = make_config(oracle_nets, cuda_device)
    files = make_files()
    alone = HyperParameterSweep(cfg)
    plain = DatasetSweep(cfg, files, sweep=alone)
    # realistic centroids: the final state the unseeded clustering holds for file 2 (5 speakers) at the config's values
    r = plain.sweep(trial_params([{}], cfg), keep_state=True)
    state = r.centers[2, 0].cpu().numpy()
    pool = state[np.einsum("md,md->m", state, state) > 0]
    assert len(pool) >= 4, f"only {len(pool)} speakers in the learned state"
    known = known_speakers(pool)
    ds = DatasetSweep(cfg, files, sweep=alone, speakers=known)
    runs = ds.run(TRIALS)
    return cfg, files, alone, plain, known, ds, runs


def seeded_pipeline_prediction(config, fw, uri, known):
    """Benchmark.run_single with a SpeakerDiarization seeded with ``known``: batches of 256, shift = -left padding"""
    pipe = blocks.SpeakerDiarization(config)
    pipe.set_known_speakers(known)
    pipe.set_timestamp_shift(-fw.padding[0])
    acc = PredictionAccumulator(uri)
    sr = config.sample_rate
    chunks = [SlidingWindowFeature(fw.window(i)[:, None], SlidingWindow(start=fw.starts[i], duration=1 / sr, step=1 / sr))
              for i in range(fw.num_windows)]
    for i in range(0, len(chunks), 256):
        for out in pipe(chunks[i:i + 256]):
            acc.on_next(out)
    return acc.get_prediction()


def test_labels_follow_the_files(seeded):
    cfg, files, alone, plain, known, ds, runs = seeded
    assert [k is None for k in ds.speakers] == [False, True, False, False, True, False]
    assert ds.labels == [speaker_labels(k, cfg.max_speakers) for k in ds.speakers]
    named = {name for f in range(len(files)) for p in runs[f] for name in p.labels() if not name.startswith("speaker")}
    assert {"alice", "bob", "carol", "dave"} <= named, named


def test_predictions_equal_a_seeded_pipeline(seeded, oracle_nets, cuda_device):
    cfg, files, alone, plain, known, ds, runs = seeded
    params = trial_params(TRIALS, cfg)
    lines = 0
    for f in (0, 2, 5):
        uri, x, _ = files[f]
        fw = file_windows(x, cfg)
        for t in PRED_TRIALS:
            p = params[t]
            c = make_config(oracle_nets, cuda_device, tau_active=p[0], rho_update=p[1], delta_new=p[2])
            want = seeded_pipeline_prediction(c, fw, uri, known[f]).to_rttm()
            assert runs[f][t].to_rttm() == want, f"file {f} trial {t}"
            lines += want.count("\n")
    assert lines > 50


def test_clustering_equals_the_seeded_oracle(seeded):
    cfg, files, alone, plain, known, ds, runs = seeded
    params = trial_params(TRIALS, cfg)
    r = ds.sweep(params, keep_state=True)
    maps, centers = r.maps.cpu().numpy(), r.centers.cpu().numpy()
    for f in range(len(files)):
        c0, c1 = int(ds.offsets[f]), int(ds.offsets[f + 1])
        s_np, e_np = (t.cpu().numpy() for t in ds.file_outputs(f))
        for t, (tau, rho, delta) in enumerate(params):
            clu = seeded_oracle(cfg, known[f], tau_active=tau, rho_update=rho, delta_new=delta)
            want = np.stack([clu(s, e)[0] for s, e in zip(s_np, e_np)])
            assert np.array_equal(maps[t, c0:c1], want), f"file {f} trial {t}: maps"
            assert np.array_equal(centers[f, t], clu.centers), f"file {f} trial {t}: centroids"


def test_unseeded_files_keep_the_unseeded_bits_and_launches(seeded):
    lib = _lib.lib()
    cfg, files, alone, plain, known, ds, runs = seeded
    before = lib.dg_launch_count()
    want, want_total = plain.score(TRIALS)
    plain_launches = lib.dg_launch_count() - before
    before = lib.dg_launch_count()
    got, _ = ds.score(TRIALS)
    assert lib.dg_launch_count() - before == plain_launches + 1          # sweep_seed
    plain_runs = plain.run(TRIALS)
    for f in (1, 4):
        assert np.array_equal(got[f].as_array(), want[f].as_array()), f"file {f}"
        assert [p.to_rttm() for p in runs[f]] == [p.to_rttm() for p in plain_runs[f]]
    # no seeds at all (None or empty for every file): the unseeded sweep's launches and bits
    empty = KnownSpeakers([], np.zeros((0, 0)))
    for speakers in (None, empty, [None, empty] * 3):
        none = DatasetSweep(cfg, files, sweep=alone, speakers=speakers)
        before = lib.dg_launch_count()
        got, total = none.score(TRIALS)
        assert lib.dg_launch_count() - before == plain_launches
        assert all(np.array_equal(a.as_array(), b.as_array()) for a, b in zip(got, want))
        assert np.array_equal(total.as_array(), want_total.as_array())


def swap_names(annotation, a, b):
    out = Annotation(uri=annotation.uri, modality=annotation.modality)
    for n, (s, _, label) in enumerate(annotation.itertracks(yield_label=True)):
        out[s, n] = b if label == a else a if label == b else label
    return out


def references(kind, runs, known):
    """per file the reference of one kind: the trial-0 prediction ("own"), the same with two known names swapped, names
    absent from the gallery, or 7 labels two of which carry a known name and speaker3"""
    out = []
    for f, secs in enumerate(SECONDS):
        own = runs[f][0]
        if kind == "own":
            out.append(own)
        elif kind == "swapped":
            names = known[f].names if known[f] is not None else ()
            out.append(swap_names(own, *names[:2]) if len(names) >= 2 else own)
        elif kind == "absent":
            out.append(synth_reference(60 + f, 3 + f % 4, secs, uri=f"file{f}"))
        else:
            ref = synth_reference(80 + f, 7, secs, uri=f"file{f}")
            first = known[f].names[0] if known[f] is not None and len(known[f]) else "speaker1"
            out.append(swap_names(swap_names(ref, "spk_A", first), "spk_B", "speaker3"))
    return out


_SWEEPS = {}


def scored_sweep(seeded, kind, with_uem):
    cfg, files, alone, plain, known, ds, runs = seeded
    key = (kind, with_uem)
    if key not in _SWEEPS:
        refs = references(kind, runs, known)
        _SWEEPS[key] = (DatasetSweep(cfg, [(u, x, r) for (u, x, _), r in zip(files, refs)], sweep=alone, speakers=known,
                                     uems=UEMS if with_uem else None), refs)
    return _SWEEPS[key]


def fold(per_file):
    out = per_file[0].as_array()
    for p in per_file[1:]:
        out = out + p.as_array()
    return out


@pytest.mark.parametrize("collar,skip", list(itertools.product((0.0, 0.25), (False, True))))
@pytest.mark.parametrize("with_uem", [False, True])
@pytest.mark.parametrize("kind", ["own", "swapped", "absent", "seven"])
def test_ier_components_equal_the_protocol_oracle(seeded, kind, collar, skip, with_uem):
    cfg, files, alone, plain, known, ds, runs = seeded
    sweep, refs = scored_sweep(seeded, kind, with_uem)
    per_file, total = sweep.score(TRIALS, IdentificationErrorRate(collar, skip))
    assert isinstance(total, IdentificationErrorComponents)
    for f in range(len(files)):
        uem = UEMS[f] if with_uem else None
        want = np.stack([protocol_ier_components(refs[f], p, collar, skip, uem) for p in runs[f]])
        assert np.array_equal(per_file[f].as_array(), want), f"file {f}"
    assert np.array_equal(total.as_array(), fold(per_file))
    if kind == "own":
        assert np.all(total.ier[0] == 0.0)
    if kind == "swapped":
        own, _ = scored_sweep(seeded, "own", with_uem)
        metric = DiarizationErrorRate(collar, skip)
        der_own, _ = own.score(TRIALS, metric)
        der_swapped, _ = sweep.score(TRIALS, metric)
        assert all(np.array_equal(a.as_array(), b.as_array()) for a, b in zip(der_own, der_swapped))
        assert total.ier[0] > 0


def test_ier_equals_der_under_ders_mapping(seeded):
    """reference labels renamed to the hypothesis labels DER's optimal mapping gives them: IER is DER bit for bit"""
    cfg, files, alone, plain, known, ds, runs = seeded
    refs = references("seven", runs, known)
    renamed = []
    for f, ref in enumerate(refs):
        to_ref = der_mapping(ref, runs[f][0])              # hypothesis label -> reference label
        to_hyp = {r: h for h, r in to_ref.items()}
        out = Annotation(uri=ref.uri)
        for n, (s, _, label) in enumerate(ref.itertracks(yield_label=True)):
            out[s, n] = to_hyp.get(label, f"nobody-{label}")
        renamed.append(out)
    a = DatasetSweep(cfg, [(u, x, r) for (u, x, _), r in zip(files, refs)], sweep=alone, speakers=known)
    b = DatasetSweep(cfg, [(u, x, r) for (u, x, _), r in zip(files, renamed)], sweep=alone, speakers=known)
    want, _ = a.score([TRIALS[0]], DiarizationErrorRate())
    got, _ = b.score([TRIALS[0]], IdentificationErrorRate())
    for f in range(len(files)):
        assert np.array_equal(got[f].as_array(), want[f].as_array()), f"file {f}"


def test_a_trial_alone_a_file_alone_and_file_order(seeded):
    cfg, files, alone, plain, known, ds, runs = seeded
    sweep, refs = scored_sweep(seeded, "seven", True)
    metric = IdentificationErrorRate(0.25, True)
    many = [TRIALS[i % len(TRIALS)] for i in range(300)]
    per_many, _ = sweep.score(many, metric)
    per_one, _ = sweep.score([TRIALS[2]], metric)
    want, _ = sweep.score(TRIALS, metric)
    for f in range(len(files)):
        assert np.array_equal(per_many[f].as_array()[2], per_one[f].as_array()[0])
        assert np.array_equal(per_many[f].as_array()[:len(TRIALS)], want[f].as_array())
    data = [(u, x, r) for (u, x, _), r in zip(files, refs)]
    one = DatasetSweep(cfg, [data[3]], sweep=alone, speakers=[known[3]], uems=[UEMS[3]])
    got, total = one.score(TRIALS, metric)
    assert np.array_equal(got[0].as_array(), want[3].as_array()) and np.array_equal(total.as_array(), want[3].as_array())
    assert [p.to_rttm() for p in one.run(TRIALS)[0]] == [p.to_rttm() for p in runs[3]]
    rev = DatasetSweep(cfg, data[::-1], sweep=alone, speakers=known[::-1], uems=UEMS[::-1])
    got, _ = rev.score(TRIALS, metric)
    n = len(files)
    for f in range(n):
        assert np.array_equal(got[n - 1 - f].as_array(), want[f].as_array()), f"file {f}"
    assert [[p.to_rttm() for p in r] for r in rev.run(TRIALS)[::-1]] == [[p.to_rttm() for p in r] for r in runs]


def test_latencies_and_osp_sets_compose(seeded, oracle_nets, cuda_device):
    cfg, files, alone, plain, known, ds, runs = seeded
    refs = references("seven", runs, known)[:3]
    data = [(u, x, r) for (u, x, _), r in zip(files[:3], refs)]
    metric = IdentificationErrorRate(0.25, False)
    trials = TRIALS[:4] + [TRIALS[5]]
    multi = DatasetSweep(cfg, data, latencies=[2.0], uems=UEMS[:3], speakers=known[:3])
    scores, preds = multi.score_latencies(trials, metric=metric), multi.run_latencies(trials)
    for lat in (0.5, 2.0):
        single = DatasetSweep(make_config(oracle_nets, cuda_device, latency=lat), data, uems=UEMS[:3], speakers=known[:3])
        got, want = scores[lat], single.score(trials, metric)
        assert all(np.array_equal(a.as_array(), b.as_array()) for a, b in zip(got[0], want[0])), lat
        assert [[p.to_rttm() for p in r] for r in preds[lat]] == [[p.to_rttm() for p in r] for r in single.run(trials)]
    sets = DatasetSweep(cfg, data, osp=[{"gamma": 2.0}], speakers=known[:3])
    got, _ = sets.score([dict(t, gamma=2.0) for t in trials] + trials, metric)
    g2, _ = DatasetSweep(make_config(oracle_nets, cuda_device, gamma=2.0), data, speakers=known[:3]).score(trials, metric)
    base, _ = DatasetSweep(cfg, data, sweep=alone, speakers=known[:3]).score(trials, metric)
    T = len(trials)
    for f in range(3):
        assert np.array_equal(got[f].as_array()[:T], g2[f].as_array()), f"file {f}, gamma 2"
        assert np.array_equal(got[f].as_array()[T:], base[f].as_array()), f"file {f}, config set"


def test_python_refusals_run_no_network(seeded):
    lib = _lib.lib()
    cfg, files, alone, plain, known, ds, runs = seeded
    M = int(cfg.max_speakers)
    D = ds.emb.shape[-1]
    rng = np.random.default_rng(5)
    too_many = KnownSpeakers([f"p{i}" for i in range(M + 1)], rng.standard_normal((M + 1, D)))
    cases = [
        (known[:5], "one KnownSpeakers for every file or one entry per file, 6 in all"),
        ("alice", "one KnownSpeakers for every file"),
        ([None, None, {"alice": 1}, None, None, None], "file file2: speakers entry must be KnownSpeakers or None"),
        ([None, KnownSpeakers(["x"], np.ones((1, D + 1))), None, None, None, None],
         f"file file1: the known speakers' centroids have dimension {D + 1}, the embeddings {D}"),
        ([None] * 5 + [too_many], f"file file5: {M + 1} known speakers, at most max_speakers = {M}"),
    ]
    for speakers, match in cases:
        before = lib.dg_launch_count()
        with pytest.raises(ValueError, match=match):
            DatasetSweep(cfg, files, sweep=alone, speakers=speakers)
        assert lib.dg_launch_count() == before, match


def test_setter_refusals_change_nothing_and_mismatches_never_launch(seeded):
    lib = _lib.lib()
    cfg, files, alone, plain, known, ds, runs = seeded
    ds.score(TRIALS[:2])                                      # the handle exists with the dataset's dimensions
    h = alone._h
    M, D = int(cfg.max_speakers), ds.emb.shape[-1]
    lib.dg_sweep_set_scored_regions(h, 0, None, None)
    lib.dg_sweep_set_trial_sets(h, 0, None, 0)
    good = np.ones((2, D))
    off2 = np.array([0, 1, 2], dtype=np.int32)
    assert lib.dg_sweep_set_seeds(h, 2, off2.ctypes.data, good.ctypes.data) == 0        # two files, the dataset has six
    off6 = np.array([0, 1, 1, 1, 1, 1, 2], dtype=np.int32)
    nan, zero = good.copy(), good.copy()
    nan[1, 3] = np.nan
    zero[0] = 0.0
    many = np.ones((M + 1, D))
    for offsets, centers, message in [
            (np.array([1, 1, 1, 1, 1, 1, 2], dtype=np.int32), good, "must start at 0"),
            (np.array([0, 2, 1, 1, 1, 1, 2], dtype=np.int32), good, "offsets must not decrease"),
            (np.array([0, M + 1, M + 1, M + 1, M + 1, M + 1, M + 1], dtype=np.int32), many, f"has {M + 1} centroids"),
            (off6, nan, "centroid 0 of file 5 is not finite"),
            (off6, zero, "centroid 0 of file 0 has a zero norm")]:
        assert lib.dg_sweep_set_seeds(h, 6, offsets.ctypes.data, centers.ctypes.data) == -1, message
        assert message.encode() in lib.dg_last_error(), (message, lib.dg_last_error())
    refs, _ = ds._packed(None)
    params = np.ascontiguousarray([[0.5, 0.3, 1.0]])
    comp = np.empty((len(files), 1, 5))

    def score_files():
        return lib.dg_sweep_score_files(h, ds.seg.data_ptr(), ds.emb.data_ptr(), ds.num_chunks, len(files),
                                        ds.offsets.ctypes.data, params.ctypes.data, 1, ds.plan.ctypes.data,
                                        ds.out_start.ctypes.data, ds.out_res.ctypes.data, ds.shifts.ctypes.data, 0.05,
                                        *(a.ctypes.data for a in refs), comp.ctypes.data, None, None, 0, None)

    header = np.empty((1, ds.num_chunks, 4), dtype=np.int32)
    turns = np.empty(1 << 16, dtype=np.uint32)
    n = ctypes.c_int()
    before = lib.dg_launch_count()
    assert score_files() == -1 and b"seeds are set for 2 files" in lib.dg_last_error()
    rc = lib.dg_sweep_run_files(h, ds.seg.data_ptr(), ds.emb.data_ptr(), ds.num_chunks, len(files), ds.offsets.ctypes.data,
                                params.ctypes.data, 1, ds.plan.ctypes.data, None, None, header.ctypes.data,
                                turns.ctypes.data, len(turns), ctypes.byref(n), None)
    assert rc == -1 and b"seeds are set for 2 files" in lib.dg_last_error()
    assert lib.dg_launch_count() == before
    assert lib.dg_sweep_set_seeds(h, 0, None, None) == 0
    table = np.full((2, 32), -1, dtype=np.int32)
    table[0, :2] = [0, 1]
    assert lib.dg_sweep_set_identities(h, 2, table.ctypes.data) == 0
    for entry, message in [((0, 5), M), ((1, 0), -2), ((0, 3), 0)]:
        bad = np.full((6, 32), -1, dtype=np.int32)
        bad[0, 0] = 0
        bad[entry] = message
        assert lib.dg_sweep_set_identities(h, 6, bad.ctypes.data) == -1
        want = b"given to two reference labels" if message == 0 else b"outside [-1, max_speakers"
        assert want in lib.dg_last_error(), lib.dg_last_error()
    before = lib.dg_launch_count()
    assert score_files() == -1 and b"identities are set for 2 files" in lib.dg_last_error()
    assert lib.dg_launch_count() == before
    # the Python layer sets or clears seeds and identities before every call
    got, _ = ds.score(TRIALS[:2])
    want, _ = DatasetSweep(cfg, files, sweep=alone, speakers=known).score(TRIALS[:2])
    assert all(np.array_equal(a.as_array(), b.as_array()) for a, b in zip(got, want))
