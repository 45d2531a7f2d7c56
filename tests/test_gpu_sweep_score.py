"""DER scoring of sweep trials on the device (dg_sweep_score through diart_b200.tune.HyperParameterSweep.score): the
components equal oracle/der.py on the predictions HyperParameterSweep.run returns, bit for bit; the merged hypothesis
segments equal assemble_predictions'; launch geometry and call order do not change results; bad arguments never launch."""

import numpy as np
import pytest

from diart_b200 import _lib, synth
from diart_b200.blocks.post import post_plan
from diart_b200.core import Annotation, Segment
from diart_b200.tune import (PATCH_COLLAR, DERComponents, HyperParameterSweep, file_windows, reference_arrays,
                             trial_params)
from oracle.der import der, der_components
from test_gpu_sweep import TRIALS, make_config

pytestmark = pytest.mark.gpu


def synth_reference(seed, n_speakers, duration, uri="synth"):
    """seeded turns with overlapping speech, some past both ends of the audio"""
    rng = np.random.default_rng(seed)
    ref = Annotation(uri=uri)
    n = 0
    for k in range(n_speakers):
        t = rng.uniform(-8.0, 2.0)
        while t < duration + 6.0:
            length = rng.uniform(0.3, 9.0)
            ref[Segment(t, t + length), n] = f"spk_{chr(65 + k)}"
            n += 1
            t += length + rng.uniform(0.0, 12.0)
    return ref


def oracle_rows(reference, predictions):
    return np.stack([der_components(reference, p) for p in predictions])


@pytest.fixture(scope="module")
def file_300(oracle_nets, cuda_device):
    x = synth.synth_audio(int(300.3 * 16000), seed=777, num_speakers=5)
    cfg = make_config(oracle_nets, cuda_device)
    sweep = HyperParameterSweep(cfg)
    preds = sweep.run(x, uri="synth", trials=TRIALS)
    refs = {n: synth_reference(n, n, len(x) / 16000) for n in (3, 7)}
    return x, cfg, sweep, preds, refs


@pytest.mark.parametrize("n_ref", [3, 7])
def test_components_equal_the_oracle(file_300, n_ref):
    x, cfg, sweep, preds, refs = file_300
    got = sweep.score(x, refs[n_ref], TRIALS)
    assert set(sweep.timing) == {"network", "score"}
    want = oracle_rows(refs[n_ref], preds)
    assert np.array_equal(got.as_array(), want), np.argwhere(got.as_array() != want)
    assert got.as_array()[6, 0] == 0.0 and got.as_array()[6, 1] == got.as_array()[6, 4], "tau_active = 1: all missed"
    assert len(set(got.der.tolist())) >= 5 and np.all(got.total > 100)


def _segments_equal_assemble(sweep, x, trials):
    cfg = sweep.config
    fw = file_windows(x, cfg)
    seg, emb = sweep.network_pass(fw)
    params = trial_params(trials, cfg)
    rows, labels, names = reference_arrays(synth_reference(1, 3, len(x) / 16000))
    _, _, offsets, hseg = sweep.sweep_score(seg, emb, fw, params, rows, labels, len(names), segments=True)
    offsets, hseg = offsets.cpu().numpy(), hseg.cpu().numpy()
    preds = sweep.run(x, uri="f", trials=trials)
    M, n = cfg.max_speakers, 0
    for t, pred in enumerate(preds):
        for g in range(M):
            want = sorted((s.start, s.end) for s, _, lab in pred.itertracks(yield_label=True) if lab == f"speaker{g}")
            got = [tuple(r) for r in hseg[offsets[t * M + g]:offsets[t * M + g + 1]].tolist()]
            assert got == want, f"trial {t} label {g}"
            n += len(want)
    assert n > 50


def test_hypothesis_segments_equal_assemble_predictions(file_300):
    x, cfg, sweep, preds, refs = file_300
    _segments_equal_assemble(sweep, x, TRIALS)


def test_hypothesis_segments_at_latency_2(oracle_nets, cuda_device):
    x = synth.synth_audio(int(152.3 * 16000), seed=99, num_speakers=6)
    sweep = HyperParameterSweep(make_config(oracle_nets, cuda_device, latency=2.0))
    _segments_equal_assemble(sweep, x, TRIALS[:5])


def test_own_prediction_as_reference_scores_zero(file_300):
    x, cfg, sweep, preds, refs = file_300
    for t in (0, 1, 7):
        own = Annotation(uri="synth")
        for i, (s, _, lab) in enumerate(preds[t].itertracks(yield_label=True)):
            own[s, i] = "ref_" + lab[::-1]
        got = sweep.score(x, own, TRIALS).as_array()[t]
        assert got[0] == got[1] == got[2] == 0.0 and got[3] == got[4] > 0, (t, got)


def test_launch_geometry_does_not_change_components(file_300):
    x, cfg, sweep, preds, refs = file_300
    fw = file_windows(x, cfg)
    seg, emb = sweep.network_pass(fw)
    rng = np.random.default_rng(11)
    many = np.column_stack([rng.uniform(0.3, 0.8, 300), rng.uniform(0, 1, 300), rng.uniform(0.05, 2, 300)])
    many[:len(TRIALS)] = trial_params(TRIALS, cfg)
    rows, labels, names = reference_arrays(refs[7])
    big = sweep.sweep_score(seg, emb, fw, many, rows, labels, len(names))[0]
    for t in (0, 4, 6, 137, 299):
        one = sweep.sweep_score(seg, emb, fw, many[t:t + 1], rows, labels, len(names))[0]
        assert np.array_equal(one[0], big[t]), t


def test_fewer_hypothesis_labels_than_reference_labels(oracle_nets, cuda_device):
    x = synth.synth_audio(int(152.3 * 16000), seed=5, num_speakers=6)
    sweep = HyperParameterSweep(make_config(oracle_nets, cuda_device, max_speakers=4))
    ref = synth_reference(7, 7, len(x) / 16000)
    trials = TRIALS[:6]
    got = sweep.score(x, ref, trials).as_array()
    assert np.array_equal(got, oracle_rows(ref, sweep.run(x, uri="synth", trials=trials)))


def test_several_files(oracle_nets, cuda_device):
    sweep = HyperParameterSweep(make_config(oracle_nets, cuda_device))
    files = []
    for i, secs in enumerate((61.3, 90.0, 45.7)):
        x = synth.synth_audio(int(secs * 16000), seed=300 + i, num_speakers=4)
        files.append((x, synth_reference(40 + i, 3 + 2 * i, secs)))
    per_file, total = sweep.score_files(files, TRIALS)
    assert np.array_equal(total.as_array(), per_file[0].as_array() + per_file[1].as_array() + per_file[2].as_array())
    want = sum(oracle_rows(ref, sweep.run(x, uri="synth", trials=TRIALS)) for x, ref in files)
    assert np.array_equal(total.as_array(), want)
    oracle_der = np.array([der(r) for r in want])
    assert int(np.argmin(total.der)) == int(np.argmin(oracle_der))
    assert np.array_equal(total.der, oracle_der)


def test_score_and_run_in_any_order(file_300, oracle_nets, cuda_device):
    x, cfg, sweep, preds, refs = file_300
    trials = TRIALS[:4]
    alone_score = HyperParameterSweep(cfg).score(x, refs[3], trials).as_array()
    alone_run = [p.to_rttm() for p in HyperParameterSweep(cfg).run(x, uri="synth", trials=trials)]
    s = HyperParameterSweep(cfg)
    a = s.score(x, refs[3], trials).as_array()
    b = [p.to_rttm() for p in s.run(x, uri="synth", trials=trials)]
    c = s.score(x, refs[7], trials[:2])
    d = s.score(x, refs[3], trials).as_array()
    e = [p.to_rttm() for p in s.run(x, uri="synth", trials=trials)]
    assert np.array_equal(a, alone_score) and np.array_equal(d, alone_score)
    assert b == alone_run and e == alone_run
    assert isinstance(c, DERComponents) and len(c.total) == 2


def test_argument_checks_never_launch(file_300):
    x, cfg, sweep, preds, refs = file_300
    lib = _lib.lib()
    fw = file_windows(x, cfg)
    seg, emb = sweep.network_pass(fw)
    N, F, K = seg.shape
    h, nw = sweep._handle(F, K, emb.shape[2])
    plan, out_start, out_res = post_plan(fw.starts, sweep._seg_resolution(float(fw.starts[0]), F), np.zeros(0), np.zeros(0),
                                         nw, F, cfg.step, cfg.latency)
    plan = np.ascontiguousarray(plan)
    comp = np.zeros((4, 5))

    def call(params=np.array([[0.5, 0.3, 1.0]]), T=1, n=N, start=out_start, res=out_res, shift=0.0, collar=PATCH_COLLAR,
             rows=np.array([[0.0, 1.0], [2.0, 3.0]]), labels=np.array([0, 1], np.int32), R=2, cap=0):
        rows, labels = np.ascontiguousarray(rows, np.float64), np.ascontiguousarray(labels, np.int32)
        start, res = np.ascontiguousarray(start, np.float64), np.ascontiguousarray(res, np.float64)
        params = np.ascontiguousarray(params, np.float64)
        return lib.dg_sweep_score(h, seg.data_ptr(), emb.data_ptr(), n, params.ctypes.data, T, plan.ctypes.data,
                                  start.ctypes.data, res.ctypes.data, shift, collar, rows.ctypes.data, labels.ctypes.data,
                                  len(rows), R, comp.ctypes.data, None, None, cap, None)

    assert call() == 0
    bad_time = out_start.copy()
    bad_time[3] = np.nan
    cases = {
        "T = 0": dict(T=0), "T > 65535": dict(T=65536), "N = 0": dict(n=0),
        "param not finite": dict(params=np.array([[np.nan, 0.3, 1.0]])),
        "collar < 0": dict(collar=-0.01), "collar not finite": dict(collar=np.inf), "shift not finite": dict(shift=np.nan),
        "chunk time not finite": dict(start=bad_time), "hyp_cap < 0": dict(cap=-1),
        "R > 32": dict(R=33, labels=np.array([0, 32], np.int32)),
        "label < 0": dict(labels=np.array([0, -1], np.int32)), "label >= R": dict(labels=np.array([0, 2], np.int32)),
        "row not finite": dict(rows=np.array([[0.0, np.inf], [2.0, 3.0]])),
        "row reversed": dict(rows=np.array([[1.0, 0.0], [2.0, 3.0]])),
        "row empty": dict(rows=np.array([[1.0, 1.0], [2.0, 3.0]])),
        "rows of a label unsorted": dict(rows=np.array([[2.0, 3.0], [0.0, 1.0]]), labels=np.array([0, 0], np.int32)),
        "rows of a label overlap": dict(rows=np.array([[0.0, 2.5], [2.0, 3.0]]), labels=np.array([1, 1], np.int32)),
    }
    for name, kw in cases.items():
        before = lib.dg_launch_count()
        rc = call(**kw)
        assert rc == -1 and lib.dg_launch_count() == before, name
        assert b"dg_sweep_score" in lib.dg_last_error(), name
    # touching rows of one label and rows of different labels in any order are accepted
    assert call(rows=np.array([[0.0, 2.0], [2.0, 3.0], [0.0, 1.0]]), labels=np.array([0, 0, 1], np.int32)) == 0
    assert call(rows=np.zeros((0, 2)), labels=np.zeros(0, np.int32), R=0) == 0
    assert comp[0, 4] == 0.0 and comp[0, 2] == comp[0, 1] == 0.0
