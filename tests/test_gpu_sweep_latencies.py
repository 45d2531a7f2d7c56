"""Sweeps over several latencies on the device (dg_sweep_*_latencies, dg_vad_sweep_curve_latencies through DatasetSweep /
VoiceActivitySweep with ``latencies``): the resident outputs of each unit are the bits of each latency's own network pass,
and for every latency the components and predictions are the bits a sweep built at that latency gives; one launch per
kernel whatever the number of latencies; the default path never reaches the new entry points; bad arguments never
launch."""
import ctypes

import numpy as np
import pytest
import torch

from diart_b200 import _lib, blocks, models
from diart_b200.tune import PATCH_COLLAR, DatasetSweep, VoiceActivitySweep, trial_params
from oracle import nets
from test_gpu_sweep import TRIALS, make_config
from test_gpu_sweep_dataset import make_files
from test_gpu_sweep_score import synth_reference

pytestmark = pytest.mark.gpu

LATENCIES = [0.5, 1, 2, 3.7, "max"]
VALUES = (0.5, 1.0, 2.0, 3.7, 5.0)
VAD_TRIALS = [{}, {"tau_active": 0.0}, {"tau_active": 1.0}, {"tau_active": 0.3}, {"tau_active": 0.45},
              {"tau_active": 0.7}]


@pytest.fixture(scope="module")
def sweeps(oracle_nets, cuda_device):
    """the files of test_gpu_sweep_dataset (3.2 s with left padding, 256 / 257 / 601 windows, ...): one sweep over the five
    latencies, and one DatasetSweep per latency"""
    files = make_files()
    ds = DatasetSweep(make_config(oracle_nets, cuda_device), files, latencies=LATENCIES)
    single = {lat: DatasetSweep(make_config(oracle_nets, cuda_device, latency=lat), files) for lat in VALUES}
    return files, ds, single


def assert_same_scores(got, want, what):
    per_file, total = got
    w_per_file, w_total = want
    assert len(per_file) == len(w_per_file), what
    for f, (a, b) in enumerate(zip(per_file, w_per_file)):
        assert np.array_equal(a.as_array(), b.as_array()), f"{what}: file {f}"
    assert np.array_equal(total.as_array(), w_total.as_array()), f"{what}: total"


def rttms(runs):
    return [[p.to_rttm() for p in r] for r in runs]


def test_resident_outputs_are_each_latencys_network_pass(sweeps):
    files, ds, single = sweeps
    assert ds.latencies == VALUES
    u = ds.units
    # files of at least one chunk are one unit, except for a latency whose last network batch holds 1 to 3 windows:
    # 257 and 259 windows (132.3 s at 1 and 2 s), 257 and 258 (132.8 s at 0.5 and 1 s); the 3.2 s file has a unit per
    # left padding, and its 4 windows at 3.7 s share the 7-window unit at 5 s (stream-form batches of 4 and 7)
    assert u.num_windows[:, 1].tolist() == [256, 257, 259, 262, 265] and u.num_windows[:, 0].tolist() == [1, 1, 1, 4, 7]
    assert len(set(u.unit_of[:, 1].tolist())) == 3 and u.unit_of[0, 1] == u.unit_of[3, 1] == u.unit_of[4, 1]
    assert len(set(u.unit_of[:, 2].tolist())) == 3 and u.unit_of[2, 2] == u.unit_of[4, 2]
    assert u.unit_of[3, 0] == u.unit_of[4, 0] and len(set(u.unit_of[:, 0].tolist())) == 4
    assert all(len(set(u.unit_of[:, f].tolist())) == 1 for f in (3, 4, 5))
    assert len(ds.offsets) - 1 == 13
    for lat in VALUES:
        for f in range(len(files)):
            seg, emb = ds.file_outputs(f, lat)
            w_seg, w_emb = single[lat].file_outputs(f)
            assert torch.equal(seg, w_seg) and torch.equal(emb, w_emb), f"latency {lat}, file {f}"


def test_components_and_predictions_equal_each_latency_alone(sweeps):
    files, ds, single = sweeps
    got = ds.score_latencies(TRIALS)
    assert list(got) == list(VALUES)
    runs = ds.run_latencies(TRIALS)
    for lat in VALUES:
        assert_same_scores(got[lat], single[lat].score(TRIALS), f"latency {lat}")
        assert rttms(runs[lat]) == rttms(single[lat].run(TRIALS)), f"latency {lat}"
    # a selection, "max" by name: the same bits
    part = ds.score_latencies(TRIALS[:4], ["max", 1.0])
    assert list(part) == [1.0, 5.0]
    for lat in (1.0, 5.0):
        assert_same_scores(part[lat], single[lat].score(TRIALS[:4]), f"latency {lat} (selection)")
    assert sum(r.count("\n") for lat in VALUES for rr in rttms(runs[lat]) for r in rr) > 500


def stage(net, x, hop, st, w=None):
    """the production forward of one network through its stage hook (dg_seg_debug_stage / dg_emb_debug_stage) -> (the
    stage's map as float32 (B or B K, ...), the paths taken)"""
    B, S = x.shape
    dims = (ctypes.c_int * 4)()
    out = np.empty(B * 3 * 512, np.float32)
    lib = _lib.lib()
    if isinstance(net, models.B200PyanNet):
        rc = lib.dg_seg_debug_stage(net.handle, x.data_ptr(), B, S, hop, st, out.ctypes.data, out.size, dims)
    else:
        rc = lib.dg_emb_debug_stage(net.handle, x.data_ptr(), w.data_ptr(), B, S, w.shape[1], w.shape[2], hop, st,
                                    out.ctypes.data, out.size, dims)
    _lib.check(rc)
    return out[:dims[0] * dims[1] * dims[2]].reshape(dims[0], -1), dims[3]


def test_network_bits_and_the_batch_length(oracle_nets, cuda_device):
    """What LatencyUnits relies on, on the production forward of both networks with the pipeline's hop hint: a window's
    scores and embedding are the same bits in every batch of 4 or more consecutive windows (the sinc front end's stream
    form), and in every batch of 1 to 3 (its per-window form, as without a hint); the two forms differ.  run_sinc_prep
    (csrc/api_seg.cu) picks the form by batch length."""
    from diart_b200 import synth
    seg = models.B200PyanNet(oracle_nets[0].state_dict()).to(cuda_device)
    emb = models.B200XVectorSincNet(oracle_nets[1].state_dict()).to(cuda_device)
    S, hop = 80000, 8000
    stream = synth.synth_audio(S + hop * 255, seed=77)
    x = torch.from_numpy(synth.windows(stream, 256, chunk=S, step=hop)).float().to(cuda_device).contiguous()
    w = torch.rand(256, 293, 3, generator=torch.Generator().manual_seed(0)).to(cuda_device)
    full = {(name, h): stage(net, x, h, st, w if name == "emb" else None)
            for name, net, st in (("seg", seg, 10), ("emb", emb, 12)) for h in (hop, 0)}
    for name, net, st in (("seg", seg, 10), ("emb", emb, 12)):
        rows = full[(name, hop)][0].shape[0] // 256
        for B in (1, 2, 3, 4, 5, 7, 10, 100):
            got, paths = stage(net, x[:B].contiguous(), hop, st, w[:B].contiguous() if name == "emb" else None)
            form = hop if B >= 4 else 0
            assert bool(paths & 1) == (B >= 4), (name, B, paths)
            assert np.array_equal(got, full[(name, form)][0][:B * rows]), (name, B)
        a, b = full[(name, hop)][0][:3 * rows], full[(name, 0)][0][:3 * rows]
        assert not np.array_equal(a, b), f"{name}: the two forms of the sinc front end now agree; LatencyUnits can share more"


def test_seven_label_references_and_four_speakers(oracle_nets, cuda_device):
    files = [(uri, x, synth_reference(70 + i, 7, len(x) / 16000, uri=uri)) for i, (uri, x, _) in
             enumerate(make_files()[:4])]
    ds = DatasetSweep(make_config(oracle_nets, cuda_device, max_speakers=4), files, latencies=LATENCIES)
    trials = TRIALS[:6]
    got, runs = ds.score_latencies(trials), ds.run_latencies(trials)
    for lat in VALUES:
        alone = DatasetSweep(make_config(oracle_nets, cuda_device, max_speakers=4, latency=lat), files)
        assert_same_scores(got[lat], alone.score(trials), f"latency {lat}")
        assert rttms(runs[lat]) == rttms(alone.run(trials)), f"latency {lat}"


def vad_config(state, device, powerset=None, **kw):
    return blocks.VoiceActivityDetectionConfig(
        segmentation=models.SegmentationModel(models.B200SegmentationLoader(state, powerset=powerset)), device=device, **kw)


@pytest.mark.parametrize("powerset", [None, (3, 2)])
def test_voice_activity_equals_each_latency_alone(powerset, oracle_nets, cuda_device):
    files = make_files()
    state = oracle_nets[0].state_dict() if powerset is None else nets.make_powerset_segmentation().state_dict()
    vs = VoiceActivitySweep(vad_config(state, cuda_device, powerset, latency=2.0), files, latencies=LATENCIES)
    assert vs.latencies == VALUES
    got, runs = vs.score_latencies(VAD_TRIALS), vs.run_latencies(VAD_TRIALS)
    for lat in VALUES:
        alone = VoiceActivitySweep(vad_config(state, cuda_device, powerset, latency=lat), files)
        for f in range(len(files)):
            assert torch.equal(vs.file_outputs(f, lat), alone.file_outputs(f)), f"latency {lat}, file {f}"
        assert_same_scores(got[lat], alone.score(VAD_TRIALS), f"latency {lat}")
        assert rttms(runs[lat]) == rttms(alone.run(VAD_TRIALS)), f"latency {lat}"
        if lat == 2.0:                                     # score / run: the config's latency
            assert_same_scores(vs.score(VAD_TRIALS), alone.score(VAD_TRIALS), "score")
            assert rttms(vs.run(VAD_TRIALS)) == rttms(alone.run(VAD_TRIALS))


def test_one_launch_per_kernel_whatever_the_number_of_latencies(sweeps, oracle_nets, cuda_device):
    files, _, single = sweeps
    lib = _lib.lib()
    cfg = make_config(oracle_nets, cuda_device)
    deltas = []
    for lats in ([], LATENCIES):
        ds = DatasetSweep(cfg, files[1:4], latencies=lats)
        ds.score_latencies(TRIALS)                         # first use: buffers sized
        before = lib.dg_launch_count()
        ds.score_latencies(TRIALS)
        deltas.append(lib.dg_launch_count() - before)
    assert deltas[0] == deltas[1] > 0
    # the clustering of each (unit, trial) is each latency's own clustering over the prefix
    params = trial_params(TRIALS, cfg)
    r = ds.sweep_latencies(params, keep_maps=True)
    maps = r.maps
    for lat in VALUES:
        alone = DatasetSweep(make_config(oracle_nets, cuda_device, latency=lat), files[1:4])
        want = alone.sweep(params, keep_state=True).maps
        for f in range(3):
            c0, c1 = ds._chunk_range(f, lat)
            assert torch.equal(maps[:, c0:c1], want[:, int(alone.offsets[f]):int(alone.offsets[f + 1])]), (lat, f)


def test_the_default_path_never_reaches_the_new_entry_points(sweeps, oracle_nets, cuda_device, monkeypatch):
    files, ds, single = sweeps
    want = single[0.5].score(TRIALS)
    want_run = rttms(single[0.5].run(TRIALS))
    assert_same_scores(ds.score(TRIALS), want, "score of a sweep built with latencies")
    assert rttms(ds.run(TRIALS)) == want_run
    lib = _lib.lib()

    def refuse(*args):
        raise AssertionError("a latency entry point was called")

    for name in ("dg_sweep_run_latencies", "dg_sweep_score_latencies", "dg_vad_sweep_curve_latencies"):
        monkeypatch.setattr(lib, name, refuse)
    plain = DatasetSweep(make_config(oracle_nets, cuda_device), files)
    assert_same_scores(plain.score(TRIALS), single[0.5].score_latencies(TRIALS)[0.5], "plain")
    plain.run(TRIALS[:2])
    plain.sweep(trial_params(TRIALS, plain.config))
    VoiceActivitySweep(vad_config(oracle_nets[0].state_dict(), cuda_device), files[:2]).score(VAD_TRIALS)


def test_refusals_never_launch(sweeps):
    files, ds, _ = sweeps
    lib = _lib.lib()
    before = lib.dg_launch_count()
    with pytest.raises(ValueError, match="not constructed"):
        ds.score_latencies(TRIALS, [1.5])
    with pytest.raises(ValueError, match="not constructed"):
        ds.run_latencies(TRIALS, [0.5, 4.0])
    with pytest.raises(ValueError, match="latency"):
        ds.score_latencies([{"latency": 2.0}])
    with pytest.raises(ValueError, match="latency"):
        ds.score([{"tau_active": 0.5, "latency": 1.0}])
    assert lib.dg_launch_count() == before
    # at the ABI: virtual files that are not a prefix of one unit
    N, F, K = ds.seg.shape
    h, _ = ds._sweep._handle(F, K, ds.emb.shape[2], ds.units.nw)
    tabs = ds._tables(ds._selection(None))
    vchunk, voff, plan, out_start, out_res, shifts = tabs
    refs = ds._pack_references(ds.references * len(VALUES))
    params = np.array([[0.5, 0.3, 1.0]])
    comp = np.zeros((len(voff) - 1, 1, 5))
    header = np.zeros((1, len(vchunk), 4), np.int32)
    turns = np.zeros(1 << 16, np.uint32)
    n = ctypes.c_int()

    def call(vc, entry):
        vc = np.ascontiguousarray(vc, dtype=np.int32)
        layout = (ds.units.num_chunks, len(ds.offsets) - 1, ds.offsets.ctypes.data, len(vc), len(voff) - 1, vc.ctypes.data,
                  voff.ctypes.data, params.ctypes.data, 1, plan.ctypes.data)
        if entry == "score":
            return lib.dg_sweep_score_latencies(h, ds.seg.data_ptr(), ds.emb.data_ptr(), *layout, out_start.ctypes.data,
                                                out_res.ctypes.data, shifts.ctypes.data, PATCH_COLLAR,
                                                *(a.ctypes.data for a in refs), comp.ctypes.data, None)
        return lib.dg_sweep_run_latencies(h, ds.seg.data_ptr(), ds.emb.data_ptr(), *layout, None, header.ctypes.data,
                                          turns.ctypes.data, len(turns), ctypes.byref(n), None)

    assert call(vchunk, "score") == 0
    f_long = 3                                              # the 601-window file, one unit
    v = len(files) * (len(VALUES) - 1) + f_long             # its virtual file at 5 s
    shifted = vchunk.copy()
    shifted[voff[v]:voff[v + 1]] += 1                       # starts one chunk in and runs into the next unit
    into_next = vchunk.copy()
    v0 = f_long                                             # its virtual file at 0.5 s ...
    short_unit = int(ds.offsets[ds.units.unit_of[0, 0]])    # ... moved to the one-window unit of the 3.2 s file at 0.5 s
    into_next[voff[v0]:voff[v0 + 1]] = short_unit + np.arange(voff[v0 + 1] - voff[v0])
    for vc, message in ((shifted, b"does not start at the first chunk of a unit"), (into_next, b"crosses into the next unit")):
        for entry in ("score", "run"):
            before = lib.dg_launch_count()
            assert call(vc, entry) == -1, (message, entry)
            assert lib.dg_launch_count() == before, (message, entry)
            assert message in lib.dg_last_error(), (message, entry)
