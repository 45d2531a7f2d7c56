"""Sweeps over overlap-aware weightings on the device (DatasetSweep(..., osp=...), dg_pipeline_nets_sets and
dg_sweep_set_trial_sets): one network pass computes the scores once and the embeddings of every OSP set (gamma, beta,
normalize_embedding_weights); for every set the resident embeddings, maps, centroids, predictions and DER components are the
bits a sweep whose config has that set's values gives, whatever the other sets, their order and the number of trials; bad
arguments never launch."""
import ctypes

import numpy as np
import pytest
import torch

from diart_b200 import _lib, blocks, models, synth
from diart_b200.tune import (DatasetSweep, DiarizationErrorRate, HyperParameterSweep, file_windows, osp_dict, osp_sets,
                             trial_params)
from oracle.clustering import OracleClustering
from test_gpu_sweep import TRIALS, make_config
from test_gpu_sweep_dataset import make_files
from test_gpu_sweep_score import oracle_rows, synth_reference

pytestmark = pytest.mark.gpu

# the default (3, 10); the gamma = 2 / 1 fast paths and powf; a saturated softmax; beta = 0; min-max normalisation
SETS = [{}, {"gamma": 2}, {"gamma": 1}, {"gamma": 2.5, "beta": 7}, {"beta": 30}, {"beta": 0},
        {"normalize_embedding_weights": True}]
PARAMS = ("tau_active", "rho_update", "delta_new")


def with_set(trial, s):
    out = dict(trial)
    out.update(s)
    return out


def mixed_trials(n):
    """n trials spread over the sets, each with the tau / rho / delta of a TRIALS row"""
    return [with_set(TRIALS[i % len(TRIALS)], SETS[(i * 5 + i // len(SETS)) % len(SETS)]) for i in range(n)]


def split(trials):
    """-> {set index: (positions in trials, the trials without their OSP keys)}"""
    out = {}
    for i, t in enumerate(trials):
        g = next(g for g, s in enumerate(SETS) if all(t.get(k) == v for k, v in s.items()) and
                 all(k in s for k in t if k not in PARAMS))
        pos, rest = out.setdefault(g, ([], []))
        pos.append(i)
        rest.append({k: v for k, v in t.items() if k in PARAMS})
    return out


@pytest.fixture(scope="module")
def osp(oracle_nets, cuda_device):
    cfg = make_config(oracle_nets, cuda_device)
    files = make_files()
    ds = DatasetSweep(cfg, files, osp=SETS[1:])
    cfgs = [make_config(oracle_nets, cuda_device, **s) for s in SETS]
    alone = [HyperParameterSweep(c) for c in cfgs]
    single = [DatasetSweep(c, files, sweep=a) for c, a in zip(cfgs, alone)]
    return cfg, files, ds, cfgs, alone, single


def test_sets_are_the_constructed_ones(osp):
    cfg, files, ds, *_ = osp
    assert len(ds.osp_sets) == len(SETS)
    assert ds.osp_sets[0] == (3.0, 10.0, False) and ds.osp_sets[6] == (3.0, 10.0, True)
    N, F, K = ds.seg.shape
    assert ds.embs.shape == (len(SETS), N, K, ds.emb.shape[2]) and ds.emb.data_ptr() == ds.embs.data_ptr()
    assert ds.resident_bytes == N * (F * K + len(SETS) * K * ds.emb.shape[2]) * 4


def test_scores_and_embeddings_equal_each_sets_pipeline(osp):
    cfg, files, ds, cfgs, alone, single = osp
    assert torch.equal(ds.seg, single[0].seg)
    for g in range(len(SETS)):
        assert torch.equal(ds.seg, single[g].seg), g
        assert torch.equal(ds.embs[g], single[g].emb), f"set {g}"
    for f in (0, 2, 3):                                   # one window with left padding; 257 windows; 601 windows
        for g in (1, 3, 6):
            seg, emb = alone[g].network_pass(file_windows(files[f][1], cfg))
            got_seg, got_emb = ds.file_outputs(f, osp=SETS[g])
            assert torch.equal(got_seg, seg) and torch.equal(got_emb, emb), (f, g)
    assert not torch.equal(ds.embs[0], ds.embs[1]) and not torch.equal(ds.embs[0], ds.embs[6])


def test_scoring_and_runs_equal_each_sets_sweep(osp):
    cfg, files, ds, cfgs, alone, single = osp
    trials = mixed_trials(3 * len(SETS))
    per_file, total = ds.score(trials)
    runs = ds.run(trials)
    for g, (pos, rest) in split(trials).items():
        want, _ = single[g].score(rest)
        want_run = single[g].run(rest)
        for f in range(len(files)):
            assert np.array_equal(per_file[f].as_array()[pos], want[f].as_array()), (f, g)
            assert [runs[f][i].to_rttm() for i in pos] == [p.to_rttm() for p in want_run[f]], (f, g)
    for f, (uri, x, ref) in enumerate(files):              # and the host oracle on those predictions
        assert np.array_equal(per_file[f].as_array(), oracle_rows(ref, runs[f])), f"file {f}"
    # HyperParameterSweep.run builds its sets from the trials: the same predictions for one file
    uri, x, _ = files[4]
    assert [p.to_rttm() for p in alone[0].run(x, uri=uri, trials=trials)] == [p.to_rttm() for p in runs[4]]


def test_clustering_equals_the_oracle_on_each_sets_embeddings(osp):
    cfg, files, ds, *_ = osp
    trials = mixed_trials(len(SETS) + 3)
    rows = ds._rows(trials)
    r = ds.sweep(rows, keep_state=True)
    maps, centers = r.maps.cpu().numpy(), r.centers.cpu().numpy()
    for f in (0, 2, 4):
        c0, c1 = int(ds.offsets[f]), int(ds.offsets[f + 1])
        s_np = ds.seg[c0:c1].cpu().numpy()
        for t, (tau, rho, delta, g) in enumerate(rows):
            e_np = ds.embs[int(g), c0:c1].cpu().numpy()
            replay = OracleClustering(tau, rho, delta, "cosine", cfg.max_speakers)
            want = np.stack([replay(s, e)[0] for s, e in zip(s_np, e_np)])
            assert np.array_equal(maps[t, c0:c1], want), f"file {f} trial {t}: maps"
            assert np.array_equal(centers[f, t], replay.centers), f"file {f} trial {t}: centroids"


def test_one_trial_alone_equals_it_among_300(osp):
    """300 trials x 6 files = 1800 states over 7 sets: several waves of the clustering launch"""
    cfg, files, ds, *_ = osp
    rng = np.random.default_rng(23)
    many = [with_set(dict(zip(PARAMS, p)), SETS[int(rng.integers(len(SETS)))]) for p in
            np.column_stack([rng.uniform(0.3, 0.8, 300), rng.uniform(0, 1, 300), rng.uniform(0.05, 2, 300)]).tolist()]
    big, _ = ds.score(many)
    for t in (0, 5, 77, 299):
        small, _ = ds.score(many[t:t + 1])
        for f in range(len(files)):
            assert np.array_equal(small[f].as_array()[0], big[f].as_array()[t]), (f, t)


def test_permuted_sets_permute_only_the_layout(osp):
    cfg, files, ds, *_ = osp
    perm = DatasetSweep(cfg, files[:3], osp=SETS[:0:-1])
    assert perm.osp_sets == (ds.osp_sets[0],) + ds.osp_sets[:0:-1]
    for g, s in enumerate(SETS):
        for f in range(3):
            assert torch.equal(perm.file_outputs(f, osp=s)[1], ds.file_outputs(f, osp=s)[1]), (f, g)
    trials = mixed_trials(2 * len(SETS))
    a, _ = perm.score(trials)
    b, _ = ds.score(trials)
    assert all(np.array_equal(a[f].as_array(), b[f].as_array()) for f in range(3))


def test_latencies_and_a_scoring_protocol_compose(osp, oracle_nets, cuda_device):
    cfg, files, ds, cfgs, *_ = osp
    sub = files[:3]
    uems = [[(1.0, len(x) / 16000 - 1.0)] for _, x, _ in sub]
    metric = DiarizationErrorRate(collar=0.25, skip_overlap=True)
    both = DatasetSweep(cfg, sub, latencies=[2.0], uems=uems, osp=SETS[3:5])
    trials = [with_set(TRIALS[i], SETS[[0, 3, 4][i % 3]]) for i in range(9)]
    got = both.score_latencies(trials, metric=metric)
    got_default = both.score_latencies(trials)
    for g, (pos, rest) in split(trials).items():
        one = DatasetSweep(cfgs[g], sub, latencies=[2.0], uems=uems)
        for want_all, have in ((one.score_latencies(rest, metric=metric), got), (one.score_latencies(rest), got_default)):
            for lat in both.latencies:
                for f in range(len(sub)):
                    assert np.array_equal(have[lat][0][f].as_array()[pos], want_all[lat][0][f].as_array()), (g, lat, f)


def test_the_configs_own_set_keeps_the_bits_and_the_launches(osp):
    cfg, files, ds, cfgs, alone, single = osp
    lib = _lib.lib()
    counts = []
    for kw in ({}, {"osp": [{}, {"gamma": 3.0, "beta": 10.0}]}):
        before = lib.dg_launch_count()
        d = DatasetSweep(cfg, files[:2], sweep=alone[0], **kw)
        d.score(TRIALS[:4])
        counts.append(lib.dg_launch_count() - before)
        per_file, _ = d.score(TRIALS[:4])
        assert len(d.osp_sets) == 1 and d.embs.shape[0] == 1
        assert all(np.array_equal(per_file[f].as_array(), single[0].score(TRIALS[:4])[0][f].as_array()) for f in range(2))
    assert counts[0] == counts[1]
    # HyperParameterSweep.score with gamma in the trials equals the dataset row
    uri, x, ref = files[5]
    trials = [with_set(TRIALS[1], SETS[1]), with_set(TRIALS[2], SETS[5]), TRIALS[3]]
    got = alone[0].score(x, ref, trials).as_array()
    per_file, _ = ds.score(trials)
    assert np.array_equal(got, per_file[5].as_array())
    per_file, _ = alone[0].score_files([(x, ref)], trials)
    assert np.array_equal(got, per_file[0].as_array())


def test_wespeaker_embedding(cuda_device, oracle_nets):
    from oracle import nets

    seg_o = oracle_nets[0]
    wespeaker = nets.make_wespeaker()

    def config(**kw):
        return blocks.SpeakerDiarizationConfig(
            segmentation=models.SegmentationModel(models.B200SegmentationLoader(seg_o.state_dict())),
            embedding=models.EmbeddingModel(models.B200EmbeddingLoader(wespeaker.state_dict())), device=cuda_device, **kw)

    files = [(f"w{i}", synth.synth_audio(int(s * 16000), seed=300 + i, num_speakers=3),
              synth_reference(90 + i, 3, s, uri=f"w{i}")) for i, s in enumerate((9.3, 31.7))]
    sets = [{}, {"gamma": 2, "beta": 5}, {"normalize_embedding_weights": True}]
    ds = DatasetSweep(config(), files, osp=sets[1:])
    trials = [with_set(TRIALS[i], sets[i % 3]) for i in range(6)]
    per_file, _ = ds.score(trials)
    for g, s in enumerate(sets):
        one = DatasetSweep(config(**s), files)
        assert torch.equal(ds.embs[g], one.emb), g
        pos = [i for i in range(6) if i % 3 == g]
        want, _ = one.score([{k: v for k, v in trials[i].items() if k in PARAMS} for i in pos])
        assert all(np.array_equal(per_file[f].as_array()[pos], want[f].as_array()) for f in range(2)), g


def test_refusals_never_launch(osp):
    cfg, files, ds, cfgs, alone, _ = osp
    lib = _lib.lib()
    before = lib.dg_launch_count()
    with pytest.raises(ValueError, match="was not constructed") as e:
        ds.score([TRIALS[1], {"gamma": 4}])
    assert "'gamma': 2.0" in str(e.value) and "trial 1" in str(e.value)
    with pytest.raises(ValueError, match="was not constructed"):
        ds.file_outputs(0, osp={"beta": 11})
    assert lib.dg_launch_count() == before
    # the handle's trial sets against the next call's T, and indices out of range
    N, F, K = ds.seg.shape
    h, _ = alone[0]._handle(F, K, ds.emb.shape[2])
    header = np.zeros((2, N, 4), np.int32)
    turns = np.zeros(1 << 20, np.uint32)
    n = ctypes.c_int()
    params = np.ascontiguousarray(trial_params(TRIALS[:2], cfg))

    def run(T):
        return lib.dg_sweep_run_files(h, ds.seg.data_ptr(), ds.embs.data_ptr(), N, len(files), ds.offsets.ctypes.data,
                                      params.ctypes.data, T, ds.plan.ctypes.data, None, None, header.ctypes.data,
                                      turns.ctypes.data, len(turns), ctypes.byref(n), None)

    idx = np.array([0, 6], np.int32)
    assert lib.dg_sweep_set_trial_sets(h, len(SETS), idx.ctypes.data, 2) == 0
    before = lib.dg_launch_count()
    assert run(1) == -1 and lib.dg_launch_count() == before
    assert b"dg_sweep_run_files" in lib.dg_last_error()
    bad = np.array([0, 7], np.int32)
    assert lib.dg_sweep_set_trial_sets(h, len(SETS), bad.ctypes.data, 2) == -1
    assert lib.dg_sweep_set_trial_sets(h, 65, idx.ctypes.data, 2) == -1
    assert lib.dg_sweep_set_trial_sets(h, 0, None, 0) == 0
    # dg_pipeline_nets_sets: bad sizes, and submitted steps outstanding
    pipe = blocks.SpeakerDiarization(cfg)
    x = torch.from_numpy(synth.windows(synth.synth_audio(80000 + 8000, seed=5), 2)).to(ds.seg.device)
    hp, F, K, D = pipe._ensure_fused(x.shape[1])
    seg = torch.empty((2, F, K), device=x.device)
    emb = torch.empty((2, 2, K, D), device=x.device)
    osp_rows = np.array([[3, 10], [2, 5]], np.float32)
    norm = np.zeros(2, np.int32)

    def nets(B=2, G=2, stride=2 * K * D, rows=osp_rows, nm=norm):
        return lib.dg_pipeline_nets_sets(hp, x.data_ptr(), B, x.shape[1], G, rows.ctypes.data, nm.ctypes.data,
                                         seg.data_ptr(), emb.data_ptr(), stride, None)

    before = lib.dg_launch_count()
    for kw in (dict(B=0), dict(G=0), dict(G=65), dict(stride=2 * K * D - 1), dict(rows=np.array([[np.nan, 10], [2, 5]], np.float32)),
               dict(nm=np.array([0, 2], np.int32))):
        assert nets(**kw) == -1, kw
        assert b"dg_pipeline_nets_sets" in lib.dg_last_error()
    assert lib.dg_launch_count() == before
    pipe.submit(x)
    before = lib.dg_launch_count()
    assert nets() == -1 and lib.dg_launch_count() == before
    assert b"outstanding" in lib.dg_last_error()
    pipe.collect()
    assert nets() == 0
    torch.cuda.synchronize()
    assert osp_sets(cfg, [osp_dict((2.0, 5.0, False))])[1] == (2.0, 5.0, False)
