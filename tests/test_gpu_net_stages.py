"""The default networks (PyanNet, XVectorSincNet) stage by stage against a float64 evaluation (oracle.nets.*_stages on
oracle.nets.float64_copy): the maps behind every layer come from the production forward through dg_seg_debug_stage /
dg_emb_debug_stage, in both forms of the sinc layer, at chunk lengths that take the fused and the fall-back pooling paths, on
the synthetic stream and on audio with silence, DC offset and extreme levels.

Error of a stage: max |cuda - ref64| / rms(ref64) over the whole map; a stage whose float64 reference does not vary over time
(digital silence) compares absolutely.  Every case prints it per stage next to the same measure of the float32 torch
evaluation (printed for orientation only: no assertion rests on float32 torch).

BARS: measured once on the default stream (S = 80 000, B = 17, both sinc forms; NVIDIA H100 80GB HBM3, 700 W limit), bar <= 4 x
the measured value.  Three fp16 x fp16 products keep about 2^-21 per operand, so a stage of reduction length K is expected near
2^-21 sqrt(K) of its RMS; the `expect` column is that number.  The measure is a MAXIMUM over 10^5 .. 10^7 elements against an RMS,
which alone puts it about five times above the typical element's error, and the InstanceNorms divide by a per-channel deviation
that is smaller than the map's RMS: the measured values sit 6 .. 10 x above `expect` from stage 0 on (float32 torch, printed
beside them, sits at 1.5 x).  tdnn0 is 50 x above it: its 60 inputs are the LeakyReLU'd InstanceNorm output, whose error is
already 5e-5, times a weight row whose l1 norm is several times its l2 norm.  The adversarial inputs are held to the same
bars; a stage that does not meet its bar on one input is pinned in PINS with the reason and what was measured."""
import ctypes as C

import numpy as np
import pytest
import torch

from diart_b200 import _lib, models, synth
from oracle import nets

pytestmark = pytest.mark.gpu

STREAM, POOL3, LSTM16, POOLF = 1, 2, 4, 8          # dims[3] of the hooks: the paths a call took

#        stage        measured   bar      expect (2^-21 sqrt K)   why above 10 x expect
BARS = {
    "wmean":         (1.26e-08, 5.0e-08),   # in units of the window's deviation; stream form: float32 partial sums around the pivot
    "wrstd":         (4.68e-08, 1.9e-07),
    "sinc_norm0":    (6.37e-05, 2.5e-04),   # 7.6e-6  K = 251
    "sinc_norm1":    (4.06e-05, 1.6e-04),   # 9.5e-6  K = 400
    "sinc_norm2":    (4.84e-05, 1.9e-04),   # 8.3e-6  K = 300
    "lstm0":         (7.59e-05, 3.0e-04),   # 6.6e-6  K = 60 + 128 per step
    "lstm1":         (6.80e-05, 2.7e-04),
    "lstm2":         (1.00e-04, 4.0e-04),
    "lstm3":         (1.59e-04, 6.4e-04),
    "linear0":       (5.65e-05, 2.3e-04),   # 7.6e-6  K = 256
    "linear1":       (7.49e-05, 3.0e-04),   # 5.4e-6  K = 128
    "scores":        (7.84e-05, 3.1e-04),
    "tdnn0":         (4.13e-04, 1.7e-03),   # 8.3e-6  K = 300
    "tdnn1":         (1.57e-04, 6.3e-04),   # 1.9e-5  K = 1536
    "tdnn2":         (2.28e-04, 9.1e-04),   # 1.9e-5  K = 1536
    "tdnn3":         (2.64e-04, 1.1e-03),   # 1.1e-5  K = 512
    "tdnn4":         (3.30e-04, 1.3e-03),   # 1.1e-5  K = 512
    "stats_pool":    (5.83e-05, 2.3e-04),
    "embedding":     (4.00e-04, 1.6e-03),   # 2.6e-5  K = 3000
}
SEG_STAGES = ["sinc_norm0", "sinc_norm1", "sinc_norm2", "wstats", "lstm0", "lstm1", "lstm2", "lstm3", "linear0", "linear1", "scores"]
EMB_STAGES = ["sinc_norm0", "sinc_norm1", "sinc_norm2", "wstats", "tdnn0", "tdnn1", "tdnn2", "tdnn3", "tdnn4"]
POOLED_FUSED, POOLED_PLAIN, EMB_FUSED, EMB_PLAIN = 9, 10, 11, 12


# ------------------------------------------------------------------------------------------------ inputs
def _speech(n, seed=77):
    return synth.synth_audio(n, seed=seed).astype(np.float64)


def _tone(n, hz):
    return 0.3 * np.sin(2 * np.pi * hz * np.arange(n) / 16000.0)


def _unit(x):
    return x / np.abs(x).max()


INPUTS = {
    "default": lambda n: _speech(n),
    "silence": lambda n: np.zeros(n),
    "half_silent": lambda n: np.where(np.arange(n) < 48000, 0.0, _speech(n)),
    "dc+0.5_a1e-1": lambda n: 0.5 + 1e-1 * _unit(_speech(n)),
    "dc+0.5_a1e-3": lambda n: 0.5 + 1e-3 * _unit(_speech(n)),
    "dc+0.05_a1e-1": lambda n: 0.05 + 1e-1 * _unit(_speech(n)),
    "dc+0.05_a1e-3": lambda n: 0.05 + 1e-3 * _unit(_speech(n)),
    "dc-0.5_a1e-1": lambda n: -0.5 + 1e-1 * _unit(_speech(n)),
    "dc-0.5_a1e-3": lambda n: -0.5 + 1e-3 * _unit(_speech(n)),
    "quiet_1e-4": lambda n: 1e-4 * _unit(_speech(n)),
    "clipped": lambda n: np.clip(4.0 * _unit(_speech(n)), -1.0, 1.0),
    "tone_50Hz": lambda n: _tone(n, 50.0),
    "tone_7900Hz": lambda n: _tone(n, 7900.0),
}


def make_windows(kind, B, S=80000, hop=8000):
    """B consecutive windows of one float32 stream, so that both forms of the sinc layer apply"""
    stream = INPUTS[kind](S + hop * (B - 1)).astype(np.float32)
    return torch.from_numpy(synth.windows(stream, B, chunk=S, step=hop))


# ------------------------------------------------------------------------------------------------ both sides
@pytest.fixture(scope="module")
def nets64(oracle_nets):
    seg_o, emb_o = oracle_nets
    return nets.float64_copy(seg_o), nets.float64_copy(emb_o)


@pytest.fixture(scope="module")
def cuda_nets(oracle_nets, cuda_device):
    seg_o, emb_o = oracle_nets
    return (models.B200PyanNet(seg_o.state_dict()).to(cuda_device),
            models.B200XVectorSincNet(emb_o.state_dict()).to(cuda_device))


class Hook:
    """one network's stage hook on one batch"""

    def __init__(self, net, x_dev, hop, weights=None):
        self.lib, self.net, self.x, self.hop, self.w = _lib.lib(), net, x_dev, hop, weights
        self.B, self.S = x_dev.shape
        self.is_seg = isinstance(net, models.B200PyanNet)
        self.paths = 0

    def __call__(self, stage):
        dims = (C.c_int * 4)()
        widest = self.B * (self.S // 30 + 8) * 80 if stage < 4 else self.B * 300 * 1500
        out = np.empty(widest, np.float32)
        if self.is_seg:
            rc = self.lib.dg_seg_debug_stage(self.net.handle, self.x.data_ptr(), self.B, self.S, self.hop, stage,
                                             out.ctypes.data, out.size, dims)
        else:
            w = self.w
            rc = self.lib.dg_emb_debug_stage(self.net.handle, self.x.data_ptr(), _lib.ptr(w), self.B, self.S,
                                             w.shape[1] if w is not None else 0, w.shape[2] if w is not None else 0, self.hop,
                                             stage, out.ctypes.data, out.size, dims)
        _lib.check(rc)
        self.paths = dims[3]
        n = dims[0] * dims[1] * dims[2]
        return out[:n].reshape(dims[0], dims[1], dims[2]).astype(np.float64)


def stage_error(got, ref):
    """max |got - ref| / rms(ref); absolute where the reference is constant over time"""
    ref = np.asarray(ref, np.float64)
    assert got.shape == ref.shape, (got.shape, ref.shape)
    assert np.isfinite(got).all(), "NaN or Inf"
    constant = ref.ndim == 3 and ref.shape[1] > 1 and np.ptp(ref, axis=1).max() < 1e-12
    scale = 1.0 if constant else np.sqrt(np.mean(ref ** 2))
    return float(np.abs(got - ref).max() / scale)


def wstats_errors(got, ref):
    """the mean on the scale of the window's standard deviation, the reciprocal standard deviation relatively"""
    mean, rstd = got[0, :, 0], got[1, :, 0]
    assert np.isfinite(got).all()
    ulp = np.spacing(np.abs(ref["wmean"].numpy()).astype(np.float32)).astype(np.float64)    # the mean is kept in float32
    return {"wmean": float((np.maximum(np.abs(mean - ref["wmean"].numpy()) - ulp, 0.0) * ref["wrstd"].numpy()).max()),
            "wrstd": float(np.abs(rstd / ref["wrstd"].numpy() - 1.0).max())}


def compare(label, hook, stages, ref, ref32, rows=None):
    """-> {stage: error}; prints every stage next to float32 torch's distance from float64"""
    errs = {}
    sel = (lambda a: a) if rows is None else (lambda a: a[rows])
    for i, name in enumerate(stages):
        if name is None:
            continue
        got = hook(i)
        if name == "wstats":
            e, e32 = wstats_errors(got, ref), None
            if ref32 is not None:
                g32 = np.stack([ref32["wmean"].numpy(), ref32["wrstd"].numpy()])[:, :, None].astype(np.float64)
                e32 = wstats_errors(g32, ref)
            for k in e:
                errs[k] = e[k]
                print(f"{label:58s} {k:11s} cuda {e[k]:.2e}   torch32 {e32[k] if e32 else float('nan'):.2e}")
            continue
        errs[name] = stage_error(sel(got), sel(ref[name].numpy()))
        e32 = stage_error(sel(ref32[name].double().numpy()), sel(ref[name].numpy())) if ref32 is not None else float("nan")
        print(f"{label:58s} {name:11s} cuda {errs[name]:.2e}   torch32 {e32:.2e}")
    return errs


def assert_bars(label, errs):
    bad = {k: (v, BARS[k][1]) for k, v in errs.items() if not v <= BARS[k][1]}
    assert not bad, f"{label}: stages beyond their bar (error, bar): {bad}"


_REFS = {}


def references(key, fn):
    """float64 (and float32, for the printout) stage maps, computed once per module and input"""
    if key not in _REFS:
        _REFS[key] = fn()
    return _REFS[key]


def seg_refs(nets64, oracle_nets, kind, x, rows=None):
    xs = x if rows is None else x[rows]
    return references(("seg", kind, tuple(x.shape), None if rows is None else tuple(rows)), lambda: (
        nets.segmentation_stages(nets64[0], xs[:, None, :].double()), nets.segmentation_stages(oracle_nets[0], xs[:, None, :])))


def emb_refs(nets64, oracle_nets, kind, x, w=None, tag=""):
    return references(("emb", kind, tuple(x.shape), tag), lambda: (
        nets.embedding_stages(nets64[1], x[:, None, :].double(), None if w is None else w.double()),
        nets.embedding_stages(oracle_nets[1], x[:, None, :], w)))


# ------------------------------------------------------------------------------------------------ shapes and paths
SHAPES = [   # S, B, fused MaxPool3 in conv1 / conv2
    (80000, 5, True), (80000, 17, True), (80000, 1, True), (48000, 5, False), (32000, 5, False)]


@pytest.mark.parametrize("hop", [8000, 0], ids=["stream", "window"])
@pytest.mark.parametrize("S,B,pool3", SHAPES)
def test_segmentation_stages(nets64, oracle_nets, cuda_nets, cuda_device, S, B, pool3, hop):
    x = make_windows("default", B, S)
    ref, ref32 = seg_refs(nets64, oracle_nets, "default", x)
    hook = Hook(cuda_nets[0], x.to(cuda_device), hop)
    label = f"seg default S={S} B={B} {'stream' if hop else 'window'}"
    errs = compare(label, hook, SEG_STAGES, ref, ref32)
    assert bool(hook.paths & STREAM) == (hop > 0 and B >= 4), "sinc form"
    assert bool(hook.paths & POOL3) == pool3, "MaxPool3 path"
    assert not hook.paths & LSTM16
    assert_bars(label, errs)


@pytest.mark.parametrize("hop", [8000, 0], ids=["stream", "window"])
@pytest.mark.parametrize("S,B,pool3", SHAPES)
def test_embedding_trunk_stages(nets64, oracle_nets, cuda_nets, cuda_device, S, B, pool3, hop):
    x = make_windows("default", B, S)
    ref, ref32 = emb_refs(nets64, oracle_nets, "default", x)
    hook = Hook(cuda_nets[1], x.to(cuda_device), hop)
    label = f"emb default S={S} B={B} {'stream' if hop else 'window'}"
    errs = compare(label, hook, EMB_STAGES, ref, ref32)
    assert bool(hook.paths & STREAM) == (hop > 0 and B >= 4), "sinc form"
    assert bool(hook.paths & POOL3) == pool3, "MaxPool3 path"
    got5 = hook(8)                                           # TDNN5 as float32, from the un-fused trunk
    e5 = stage_error(got5, ref["tdnn4"].numpy())
    print(f"{label:58s} {'tdnn4(f32)':11s} cuda {e5:.2e}")
    errs["tdnn4"] = max(errs["tdnn4"], e5)
    assert_bars(label, errs)


def test_wide_batch_recurrence_16_rows(nets64, oracle_nets, cuda_nets, cuda_device):
    """136 windows: the recurrence runs 16 rows per CTA with a partial last CTA; the float64 reference runs on the windows
    around the first CTA boundary and on the partial CTA only"""
    B, rows = 136, list(range(14, 19)) + list(range(128, 136))
    x = make_windows("default", B)
    ref, ref32 = seg_refs(nets64, oracle_nets, "default", x, rows)
    hook = Hook(cuda_nets[0], x.to(cuda_device), 8000)
    stages = [None, None, "sinc_norm2", None] + SEG_STAGES[4:]
    label = "seg default S=80000 B=136 stream, windows 14-18, 128-135"
    # `ref` holds only `rows`; the hook returns all windows
    errs = {}
    for i, name in enumerate(stages):
        if name is None:
            continue
        got = hook(i)[rows]
        errs[name] = stage_error(got, ref[name].numpy())
        print(f"{label:58s} {name:11s} cuda {errs[name]:.2e}   torch32 {stage_error(ref32[name].double().numpy(), ref[name].numpy()):.2e}")
    assert hook.paths & LSTM16 and hook.paths & STREAM and hook.paths & POOL3
    assert_bars(label, errs)


# ------------------------------------------------------------------------------------------------ adversarial audio
# Stages that do not meet the default stream's bar on one input, each with the reason and an upper bound just above what was
# measured (H100 80GB HBM3, 700 W).  Every other stage of the case keeps the default bar, and every stage must be finite.
_EPS = "the level is 200 x below the 1e-5 epsilon of the waveform norm, so the normalised signal is 0.003 of the constant it rides on"
_TONE = ("a pure tone leaves most filters' outputs near zero and InstanceNorm amplifies what is left; float32 torch is as far from "
         "float64 (printed beside each stage)")
PINS = {   # input: {stage: bound}, both sinc forms; measured = the larger of the two forms
    "dc-0.5_a1e-3": {"lstm1": 3.6e-4},     # measured 3.2e-4 (float32 torch 1.9e-4 on this input)
    "clipped": {"wrstd": 2.5e-7},          # measured 2.2e-7 in the per-window form: float32 partial sums of squares at full scale
    # measured 2.3e-4, 2.8e-4, 4.9e-4, 5.0e-4, 5.5e-4, 3.4e-4, 3.4e-4: _EPS
    "quiet_1e-4": {"sinc_norm1": 2.6e-4, "sinc_norm2": 3.1e-4, "lstm0": 5.4e-4, "lstm1": 5.5e-4, "lstm2": 6.0e-4, "linear0": 3.8e-4,
                   "linear1": 3.8e-4},
    # bounds 1.25 x measured: _TONE
    "tone_50Hz": {"sinc_norm0": 1.8e-3, "sinc_norm1": 4.6e-3, "sinc_norm2": 1.2e-2, "lstm0": 1.4e-2, "lstm1": 1.4e-2, "lstm2": 1.4e-2,
                  "lstm3": 1.4e-2, "linear0": 9.5e-3, "linear1": 9.5e-3, "scores": 1.2e-2, "tdnn0": 5.3e-2, "tdnn1": 2.1e-2,
                  "tdnn2": 2.4e-2, "tdnn3": 2.9e-2, "tdnn4": 3.8e-2},
    "tone_7900Hz": {"sinc_norm0": 2.2e-3, "sinc_norm1": 5.4e-3, "sinc_norm2": 1.5e-2, "lstm0": 1.4e-2, "lstm1": 3.5e-2, "lstm2": 1.9e-2,
                    "lstm3": 1.8e-2, "linear0": 1.4e-2, "linear1": 1.1e-2, "scores": 1.8e-2, "tdnn0": 2.7e-2, "tdnn1": 2.2e-2,
                    "tdnn2": 2.5e-2, "tdnn3": 2.7e-2, "tdnn4": 3.5e-2},
}


def bar_of(kind, hop, stage):
    return PINS.get(kind, {}).get(stage, BARS[stage][1])


@pytest.mark.parametrize("hop", [8000, 0], ids=["stream", "window"])
@pytest.mark.parametrize("kind", [k for k in INPUTS if k != "default"])
def test_stages_on_adversarial_audio(nets64, oracle_nets, cuda_nets, cuda_device, kind, hop):
    """both networks, every stage finite (stage_error) and inside its bar"""
    B = 5
    x = make_windows(kind, B)
    xd = x.to(cuda_device)
    form = "stream" if hop else "window"
    bad = []
    for net, stages, (ref, ref32), who in ((cuda_nets[0], SEG_STAGES, seg_refs(nets64, oracle_nets, kind, x), "seg"),
                                           (cuda_nets[1], EMB_STAGES, emb_refs(nets64, oracle_nets, kind, x), "emb")):
        hook = Hook(net, xd, hop)
        label = f"{who} {kind} B={B} {form}"
        errs = compare(label, hook, stages, ref, ref32)
        assert bool(hook.paths & STREAM) == (hop > 0), "sinc form"
        assert hook.paths & POOL3
        bad += [(label, k, v, bar_of(kind, hop, k)) for k, v in errs.items() if not v <= bar_of(kind, hop, k)]
    assert not bad, f"beyond the bar (case, stage, error, bar): {bad}"


@pytest.mark.parametrize("kind", list(INPUTS))
def test_sinc_forms_agree_at_stage_0(nets64, oracle_nets, cuda_nets, cuda_device, kind):
    """the stream form against the per-window form, at twice the stage's bar"""
    x = make_windows(kind, 5)
    xd = x.to(cuda_device)
    for who, net, ref in (("seg", cuda_nets[0], seg_refs(nets64, oracle_nets, kind, x)[0]),
                          ("emb", cuda_nets[1], emb_refs(nets64, oracle_nets, kind, x)[0])):
        a, b = Hook(net, xd, 8000), Hook(net, xd, 0)
        ga, gb = a(0), b(0)
        assert a.paths & STREAM and not b.paths & STREAM
        constant = np.ptp(ref["sinc_norm0"].numpy(), axis=1).max() < 1e-12
        e = float(np.abs(ga - gb).max()) if constant else stage_error(ga, gb)
        print(f"{who + ' ' + kind:58s} {'stream-vs-window':11s} stage 0 {e:.2e}")
        assert e <= 2 * bar_of(kind, 8000, "sinc_norm0"), (who, kind, e)


@pytest.mark.parametrize("kind", [k for k in INPUTS if k != "default"])
def test_scores_of_a_window_do_not_depend_on_the_batch(cuda_nets, cuda_device, kind):
    seg_c, B = cuda_nets[0], 5
    xd = make_windows(kind, B).to(cuda_device)
    full = seg_c(xd[:, None, :])
    assert torch.isfinite(full).all()
    for i in (0, B - 1):
        assert torch.equal(full[i], seg_c(xd[i:i + 1, None, :])[0]), f"window {i} alone differs from window {i} in the batch"


# ------------------------------------------------------------------------------------------------ statistics pooling
def _weights(B, F, K, seed=3):
    return torch.rand((B, F, K), generator=torch.Generator().manual_seed(seed)) ** 3


POOL_CASES = [  # S, K, pool mode, stages (pooled, embedding), fused
    (80000, 3, "3.1", (POOLED_FUSED, EMB_FUSED), True), (80000, 4, "3.1", (POOLED_FUSED, EMB_FUSED), True),
    (80000, 3, "3.1", (POOLED_PLAIN, EMB_PLAIN), False), (80000, 5, "3.1", (POOLED_PLAIN, EMB_PLAIN), False),
    (80000, 3, "2.1", (POOLED_FUSED, EMB_FUSED), True), (80000, 3, "2.1", (POOLED_PLAIN, EMB_PLAIN), False),
    (32000, 3, "3.1", (POOLED_PLAIN, EMB_PLAIN), False)]


@pytest.fixture(scope="module")
def emb_by_mode(oracle_nets, cuda_nets, cuda_device):
    import copy

    emb21 = copy.deepcopy(oracle_nets[1])
    emb21.stats_pool.mode = "2.1"
    return {"3.1": (oracle_nets[1], cuda_nets[1]),
            "2.1": (emb21, models.B200XVectorSincNet(emb21.state_dict(), pool_mode="2.1").to(cuda_device))}


@pytest.mark.parametrize("S,K,mode,stages,fused", POOL_CASES)
def test_pooled_statistics_and_embedding(emb_by_mode, cuda_device, S, K, mode, stages, fused):
    B = 5
    emb_o, emb_c = emb_by_mode[mode]
    x = make_windows("default", B, S)
    w = _weights(B, ((((S - 251) // 10 + 1) // 3 - 4) // 3 - 4) // 3, K)      # the segmentation's frame count at this chunk length
    ref, ref32 = references(("pool", S, K, mode), lambda: (
        nets.embedding_stages(nets.float64_copy(emb_o), x[:, None, :].double(), w.double()),
        nets.embedding_stages(emb_o, x[:, None, :], w)))
    hook = Hook(emb_c, x.to(cuda_device), 8000, w.to(cuda_device))
    label = f"emb pool S={S} K={K} mode {mode} {'fused' if fused else 'un-fused'}"
    errs = {}
    for stage, name in zip(stages, ("stats_pool", "embedding")):
        got = hook(stage).reshape(B, K, -1)
        errs[name] = stage_error(got, ref[name].numpy())
        print(f"{label:58s} {name:11s} cuda {errs[name]:.2e}   torch32 {stage_error(ref32[name].double().numpy(), ref[name].numpy()):.2e}")
        assert bool(hook.paths & POOLF) == fused, "statistics pooling path"
    if not fused and (K > 4 or S < 80000):
        with pytest.raises(ValueError):
            hook(POOLED_FUSED)                     # the fused pooling does not exist here: the hook says so, it does not fall back
    assert_bars(label, errs)


@pytest.mark.parametrize("stage,fused", [(POOLED_FUSED, True), (POOLED_PLAIN, False)])
def test_pooling_weight_edges(oracle_nets, nets64, cuda_nets, cuda_device, stage, fused):
    """the denominators v1 and v1 - v2 / v1 + eps of StatsPool at their edges: a speaker with no weight at all, one with a single
    frame above the floor, one at the 1e-8 floor of OverlappedSpeechPenalty everywhere"""
    B, K, F = 5, 4, 293
    x = make_windows("default", B)
    w = _weights(B, F, K)
    w[:, :, 0] = 0.0
    w[:, :, 1] = 1e-8
    w[:, 100, 1] = 0.5                             # one frame above the floor
    w[:, :, 2] = 1e-8
    ref = references(("pool_edges",), lambda: nets.embedding_stages(nets64[1], x[:, None, :].double(), w.double()))
    hook = Hook(cuda_nets[1], x.to(cuda_device), 8000, w.to(cuda_device))
    got = hook(stage).reshape(B, K, 3000)
    want = ref["stats_pool"].numpy()
    assert bool(hook.paths & POOLF) == fused
    assert np.isfinite(got).all()
    label = f"emb pool weight edges {'fused' if fused else 'un-fused'}"
    for k, name in ((0, "all-zero"), (2, "1e-8 floor"), (3, "random")):
        e = stage_error(got[:, k], want[:, k]) if k else float(np.abs(got[:, k] - want[:, k]).max())
        print(f"{label:58s} {name:11s} cuda {e:.2e}")
        assert e <= BARS["stats_pool"][1], (name, e)


@pytest.mark.parametrize("stage,fused", [(POOLED_FUSED, True), (POOLED_PLAIN, False)])
def test_pooling_single_frame_weight(nets64, cuda_nets, cuda_device, stage, fused):
    """one frame of weight 1: the mean is that frame; float64 gives a standard deviation of 5.8e-5 |x| that comes from
    1 + 1e-8 != 1 alone -- in float32 (pyannote's too) 1 + 1e-8 == 1 and the deviation is exactly 0"""
    B, K, F = 5, 3, 293
    x = make_windows("default", B)
    w = torch.zeros((B, F, K))
    w[:, 100, :] = 1.0                             # frame 100 of 293 is the nearest-neighbour source of exactly one of the 279 frames
    ref = references(("pool_one_frame",), lambda: nets.embedding_stages(nets64[1], x[:, None, :].double(), w.double()))
    hook = Hook(cuda_nets[1], x.to(cuda_device), 8000, w.to(cuda_device))
    got, want = hook(stage).reshape(B, K, 3000), ref["stats_pool"].numpy()
    assert bool(hook.paths & POOLF) == fused and np.isfinite(got).all()
    e_mean = stage_error(got[:, :, :1500], want[:, :, :1500])
    print(f"{'emb pool one frame ' + ('fused' if fused else 'un-fused'):58s} mean {e_mean:.2e}, max std {np.abs(got[:, :, 1500:]).max():.2e}")
    assert e_mean <= BARS["stats_pool"][1]
    assert np.all(got[:, :, 1500:] >= 0) and np.all(np.abs(got[:, :, 1500:] - want[:, :, 1500:]) <= 1e-4 * np.abs(want[:, :, :1500]).max())


def test_hooks_refuse_other_models(cuda_device):
    """a WeSpeaker (variant B) handle has none of these stages"""
    lib = _lib.lib()
    emb_b = models.B200EmbeddingLoader(nets.make_wespeaker().state_dict())().to(cuda_device)
    x = make_windows("default", 1).to(cuda_device)
    out, dims = np.empty(16, np.float32), (C.c_int * 4)()
    launches = lib.dg_launch_count()
    assert lib.dg_emb_debug_stage(emb_b.handle, x.data_ptr(), None, 1, 80000, 0, 0, 0, 0, out.ctypes.data, out.size, dims) == -1
    assert b"XVectorSincNet" in lib.dg_last_error()
    assert lib.dg_launch_count() == launches
