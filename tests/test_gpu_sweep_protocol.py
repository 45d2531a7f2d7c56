"""Scoring protocols on the device (dg_sweep_set_scored_regions / dg_vad_sweep_set_scored_regions through the ``metric`` and
``uems`` arguments of diart_b200.tune): for a forgiveness collar, skip_overlap and a uem, every (file, trial) component is
bit-identical to the protocol oracle (tests/scoring_protocol.py) on the predictions ``run()`` returns; the single-file,
dataset and latency entry points agree; the default metric keeps today's bits and launches; refusals never launch."""
import itertools

import numpy as np
import pytest

from diart_b200 import _lib
from diart_b200.core import Annotation, Segment
from diart_b200.tune import (DatasetSweep, DetectionErrorRate, DiarizationErrorRate, HyperParameterSweep,
                             VoiceActivitySweep, pack_regions)
from scoring_protocol import der_components, detection_components
from test_gpu_sweep import TRIALS, make_config
from test_gpu_sweep_dataset import SECONDS, make_files
from test_gpu_vad_sweep import TAUS, as_trials
from test_gpu_vad_sweep import make_config as make_vad_config

pytestmark = pytest.mark.gpu

COLLARS, SKIPS = (0.0, 0.25, 0.5), (False, True)


def uem_of(secs):
    """three pieces that cut through speech, and leave out the padding and the ends of the reference"""
    return [(0.5, 0.4 * secs), (Segment(0.45 * secs, 0.8 * secs)), (0.85 * secs - 0.125, secs + 1.0)]


UEMS = [uem_of(s) for s in SECONDS]


def speech(annotation):
    out = Annotation(uri=annotation.uri)
    for n, (s, _) in enumerate(annotation.itertracks()):
        out[s, n] = "speech"
    return out


@pytest.fixture(scope="module")
def diarization(oracle_nets, cuda_device):
    cfg = make_config(oracle_nets, cuda_device)
    files = make_files()
    alone = HyperParameterSweep(cfg)
    plain = DatasetSweep(cfg, files, sweep=alone)
    cut = DatasetSweep(cfg, files, sweep=alone, uems=UEMS)
    runs = plain.run(TRIALS)
    return cfg, files, alone, plain, cut, runs


@pytest.fixture(scope="module")
def vad(oracle_nets, cuda_device):
    cfg = make_vad_config(oracle_nets, cuda_device)
    files = make_files()
    plain = VoiceActivitySweep(cfg, files)
    cut = VoiceActivitySweep(cfg, files, uems=UEMS)
    runs = plain.run(as_trials(TAUS))
    return cfg, files, plain, cut, runs


def fold(per_file):
    out = per_file[0].as_array()
    for p in per_file[1:]:
        out = out + p.as_array()
    return out


@pytest.mark.parametrize("collar,skip", list(itertools.product(COLLARS, SKIPS)))
@pytest.mark.parametrize("with_uem", [False, True])
def test_der_components_equal_the_oracle(diarization, collar, skip, with_uem):
    cfg, files, alone, plain, cut, runs = diarization
    sweep = cut if with_uem else plain
    per_file, total = sweep.score(TRIALS, DiarizationErrorRate(collar, skip))
    for f, (_, _, ref) in enumerate(files):
        uem = UEMS[f] if with_uem else None
        want = np.stack([der_components(ref, p, collar, skip, uem) for p in runs[f]])
        assert np.array_equal(per_file[f].as_array(), want), f"file {f}"
    assert np.array_equal(total.as_array(), fold(per_file))


@pytest.mark.parametrize("collar,skip", list(itertools.product(COLLARS, SKIPS)))
@pytest.mark.parametrize("with_uem", [False, True])
def test_detection_components_equal_the_oracle(vad, collar, skip, with_uem):
    cfg, files, plain, cut, runs = vad
    sweep = cut if with_uem else plain
    per_file, total = sweep.score(as_trials(TAUS), DetectionErrorRate(collar, skip))
    for f, (_, _, ref) in enumerate(files):
        uem = UEMS[f] if with_uem else None
        want = np.stack([detection_components(speech(ref), p, collar, skip, uem) for p in runs[f]])
        assert np.array_equal(per_file[f].as_array(), want), f"file {f}"
    assert np.array_equal(total.as_array(), fold(per_file))


def test_one_file_sweep_equals_the_dataset_row(diarization):
    cfg, files, alone, plain, cut, runs = diarization
    metric = DiarizationErrorRate(0.25, True)
    per_file, _ = cut.score(TRIALS, metric)
    for f in (0, 3):
        _, x, ref = files[f]
        got = alone.score(x, ref, TRIALS, metric=metric, uem=UEMS[f])
        assert np.array_equal(got.as_array(), per_file[f].as_array()), f"file {f}"


def test_default_metric_keeps_the_bits_and_the_launches(diarization, vad):
    lib = _lib.lib()
    cfg, files, alone, plain, cut, runs = diarization
    outs, launches = [], []
    for metric in (None, DiarizationErrorRate(), DiarizationErrorRate(0.0, False), None):
        before = lib.dg_launch_count()
        per_file, _ = plain.score(TRIALS, metric)
        launches.append(lib.dg_launch_count() - before)
        outs.append([p.as_array() for p in per_file])
    assert len(set(launches)) == 1 and launches[0] > 0
    assert all(np.array_equal(a, b) for o in outs[1:] for a, b in zip(o, outs[0]))
    _, x, ref = files[1]
    assert np.array_equal(alone.score(x, ref, TRIALS, metric=DiarizationErrorRate()).as_array(), outs[0][1])
    vcfg, vfiles, vplain, vcut, vruns = vad
    outs, launches = [], []
    for metric in (None, DetectionErrorRate(), None):
        before = lib.dg_launch_count()
        per_file, _ = vplain.score(as_trials(TAUS), metric)
        launches.append(lib.dg_launch_count() - before)
        outs.append([p.as_array() for p in per_file])
    assert len(set(launches)) == 1 and launches[0] > 0
    assert all(np.array_equal(a, b) for o in outs[1:] for a, b in zip(o, outs[0]))


def test_a_trial_alone_equals_it_among_300_and_file_order(diarization, oracle_nets, cuda_device):
    cfg, files, alone, plain, cut, runs = diarization
    metric = DiarizationErrorRate(0.5, True)
    many = [TRIALS[i % len(TRIALS)] for i in range(300)]
    per_many, _ = cut.score(many, metric)
    per_one, _ = cut.score([TRIALS[2]], metric)
    for f in range(len(files)):
        assert np.array_equal(per_many[f].as_array()[2], per_one[f].as_array()[0])
        assert np.array_equal(per_many[f].as_array()[:len(TRIALS)], per_many[f].as_array()[len(TRIALS):2 * len(TRIALS)])
    rev = DatasetSweep(cfg, files[::-1], sweep=alone, uems=UEMS[::-1])
    per_rev, _ = rev.score(TRIALS, metric)
    want, _ = cut.score(TRIALS, metric)
    for f in range(len(files)):
        assert np.array_equal(per_rev[len(files) - 1 - f].as_array(), want[f].as_array())


def test_score_latencies_equal_each_latency_alone(oracle_nets, cuda_device):
    files = make_files()[:3]
    uems = UEMS[:3]
    metric = DiarizationErrorRate(0.25, True)
    cfg = make_config(oracle_nets, cuda_device)
    multi = DatasetSweep(cfg, files, latencies=[2.0], uems=uems).score_latencies(TRIALS[:4], metric=metric)
    for lat in (0.5, 2.0):
        single = DatasetSweep(make_config(oracle_nets, cuda_device, latency=lat), files, uems=uems).score(TRIALS[:4], metric)
        assert all(np.array_equal(a.as_array(), b.as_array()) for a, b in zip(multi[lat][0], single[0])), lat
    vmetric = DetectionErrorRate(0.5, False)
    vcfg = make_vad_config(oracle_nets, cuda_device)
    vmulti = VoiceActivitySweep(vcfg, files, latencies=[2.0], uems=uems).score_latencies(as_trials(TAUS), metric=vmetric)
    for lat in (0.5, 2.0):
        vsingle = VoiceActivitySweep(make_vad_config(oracle_nets, cuda_device, latency=lat), files,
                                     uems=uems).score(as_trials(TAUS), vmetric)
        assert all(np.array_equal(a.as_array(), b.as_array()) for a, b in zip(vmulti[lat][0], vsingle[0])), lat


def test_edge_cases(diarization, vad):
    cfg, files, alone, plain, cut, runs = diarization
    _, x, ref = files[4]
    secs = SECONDS[4]
    # every reference segment shorter than the collar: the reference is empty after the collar, total 0
    short = Annotation(uri="short")
    for n, t in enumerate(np.arange(1.0, secs - 1.0, 3.0)):
        short[Segment(t, t + 0.25), n] = f"spk{n % 3}"
    got = alone.score(x, short, TRIALS, metric=DiarizationErrorRate(0.5))
    want = np.stack([der_components(short, p, 0.5) for p in runs[4]])
    assert np.array_equal(got.as_array(), want)
    assert np.all(got.total == 0) and np.array_equal(got.der, np.where(got.false_alarm > 0, 1.0, 0.0))
    # a uem of many short pieces: hypotheses cross every edge
    comb = [(t, t + 1.5) for t in np.arange(0.0, secs, 2.0)]
    got = alone.score(x, ref, TRIALS, uem=comb)
    want = np.stack([der_components(ref, p, 0.0, False, comb) for p in runs[4]])
    assert np.array_equal(got.as_array(), want)
    vcfg, vfiles, vplain, vcut, vruns = vad
    one = VoiceActivitySweep(vcfg, [vfiles[4]], uems=[comb])
    got, _ = one.score(as_trials(TAUS), DetectionErrorRate(0.25, True))
    want = np.stack([detection_components(speech(ref), p, 0.25, True, comb) for p in vruns[4]])
    assert np.array_equal(got[0].as_array(), want)


def test_a_file_count_mismatch_never_launches(diarization, vad):
    lib = _lib.lib()
    cfg, files, alone, plain, cut, runs = diarization
    cut.score(TRIALS[:2], DiarizationErrorRate(0.25))          # the handle exists with the dataset's dimensions
    h = alone._h
    rows, off = pack_regions([[(0.0, 10.0)], [(1.0, 2.0)]])   # two files, the dataset has six
    assert lib.dg_sweep_set_scored_regions(h, 2, rows.ctypes.data, off.ctypes.data) == 0
    refs, _ = plain._packed(None)
    params = np.ascontiguousarray([[0.5, 0.3, 1.0]])
    comp = np.empty((len(files), 1, 5))
    N = plain.num_chunks
    before = lib.dg_launch_count()
    rc = lib.dg_sweep_score_files(h, plain.seg.data_ptr(), plain.emb.data_ptr(), N, len(files), plain.offsets.ctypes.data,
                                  params.ctypes.data, 1, plain.plan.ctypes.data, plain.out_start.ctypes.data,
                                  plain.out_res.ctypes.data, plain.shifts.ctypes.data, 0.05,
                                  *(a.ctypes.data for a in refs), comp.ctypes.data, None, None, 0, None)
    assert rc == -1 and lib.dg_launch_count() == before
    assert b"scored regions are set for 2 files" in lib.dg_last_error()
    vcfg, vfiles, vplain, vcut, vruns = vad
    assert lib.dg_vad_sweep_set_scored_regions(vplain._h, 2, rows.ctypes.data, off.ctypes.data) == 0
    vrefs, _ = vplain._packed(None)
    taus = np.array([0.5])
    vcomp = np.empty((len(files), 1, 2))
    before = lib.dg_launch_count()
    rc = lib.dg_vad_sweep_score_files(vplain._h, taus.ctypes.data, 1, vplain.out_start.ctypes.data,
                                      vplain.out_res.ctypes.data, vplain.shifts.ctypes.data, 0.05, vrefs[0].ctypes.data,
                                      vrefs[1].ctypes.data, vcomp.ctypes.data, None)
    assert rc == -1 and lib.dg_launch_count() == before
    # the Python layer sets or clears the regions before every call, so the sweeps still score
    a, _ = plain.score(TRIALS[:2])
    b, _ = vplain.score(as_trials(TAUS[:2]))
    assert a[0].as_array().shape == (2, 5) and b[0].as_array().shape == (2, 3)
