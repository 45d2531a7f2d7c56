"""Variant B of the embedding (WeSpeaker ResNet34) stage by stage against a float64 evaluation (oracle.nets.wespeaker_stages on
oracle.nets.float64_copy): the log-mel features, the stem and all 16 BasicBlocks come from the production trunk through
dg_emb_debug_trunk, the raw embeddings from forward_fused, at chunk lengths whose stride-2 inputs have odd and even widths, on
the synthetic stream and on audio with silence, DC offset, constant stretches and levels beyond the int16 range.

Error of a stage: max |cuda - ref64| / rms(ref64) over the whole map (tests/test_gpu_net_stages.py: stage_error, absolute
where the float64 map does not vary over time); the log-mel features compare absolutely, in the log domain.  Every case prints
float32 torch's distance from float64 beside it, for orientation only.

BARS: measured on the default stream (S = 80 000, U = 17; the embedding at U = 3, K = 3; NVIDIA H100 80GB HBM3, 700 W limit),
bar = 4 x the measured value.  Before the front end split s (x 2^15 - p) per item and floored frames of one constant value,
this file failed on the parent commit with: constant 0.5 / -0.3, log-mel 10.7 / 10.4; 3 s at 0.05 then speech, log-mel 6.9
and block15 0.85; speech at peak 6, log-mel 3.4, stem 2.8, raw embedding 1.2e-2; peak 3, stem 1.4e-3.
A stage that does not meet its bar on one input is pinned in PINS with the reason and what was measured.  (File name: the
variant-B files run after the default networks' tests.)"""
import ctypes as C

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from diart_b200 import _lib, models, synth
from oracle import nets
from test_gpu_net_stages import INPUTS, make_windows, stage_error

pytestmark = pytest.mark.gpu

STAGES = ["logmel", "stem"] + [f"block{i}" for i in range(16)]
STOP = {name: i - 2 for i, name in enumerate(STAGES)}          # dg_emb_debug_trunk's stop_after of every stage

#        stage         measured   bar       float32 torch (printed beside every case)
BARS = {
    "logmel":    (4.79e-04, 2.0e-03),   # absolute, log domain; 1.6e-4
    "stem":      (3.13e-04, 1.3e-03),   # 6.1e-5
    "block0":    (3.14e-04, 1.3e-03),
    "block1":    (2.89e-04, 1.2e-03),
    "block2":    (2.53e-04, 1.1e-03),
    "block3":    (3.09e-04, 1.3e-03),
    "block4":    (2.84e-04, 1.2e-03),
    "block5":    (2.62e-04, 1.1e-03),
    "block6":    (2.61e-04, 1.1e-03),
    "block7":    (1.36e-04, 5.5e-04),
    "block8":    (1.23e-04, 5.0e-04),
    "block9":    (1.11e-04, 4.5e-04),
    "block10":   (1.01e-04, 4.1e-04),
    "block11":   (9.49e-05, 3.8e-04),
    "block12":   (9.21e-05, 3.7e-04),
    "block13":   (7.22e-05, 2.9e-04),
    "block14":   (6.63e-05, 2.7e-04),
    "block15":   (6.90e-05, 2.8e-04),   # 2.3e-5
    "embedding": (8.37e-05, 3.4e-04),   # measured at U = 3, K = 3; 1.6e-6
}


def _speech(n, seed=77):
    return synth.synth_audio(n, seed=seed).astype(np.float64)


def _unit(x):
    return x / np.abs(x).max()


# inputs beyond those of the default networks: constant stretches at a non-zero level, and speech louder than the int16 range
B_INPUTS = {
    "const+0.5": lambda n: np.full(n, 0.5),
    "const-0.3": lambda n: np.full(n, -0.3),
    "dc+0.05_then_speech": lambda n: 0.05 + np.where(np.arange(n) < 48000, 0.0, 0.1 * _unit(_speech(n))),
    "peak3": lambda n: 3.0 * _unit(_speech(n)),
    "peak6": lambda n: 6.0 * _unit(_speech(n)),
}
ALL_INPUTS = {**INPUTS, **B_INPUTS}


def windows(kind, U, S=80000, hop=8000):
    if kind in INPUTS:
        return make_windows(kind, U, S, hop)
    stream = B_INPUTS[kind](S + hop * (U - 1)).astype(np.float32)
    return torch.from_numpy(synth.windows(stream, U, chunk=S, step=hop))


# ------------------------------------------------------------------------------------------------ both sides
@pytest.fixture(scope="module")
def wespeaker():
    torch.set_num_threads(16)
    return nets.make_wespeaker()


@pytest.fixture(scope="module")
def net64(wespeaker):
    return nets.float64_copy(wespeaker)


@pytest.fixture(scope="module")
def emb_b(wespeaker, cuda_device):
    return models.B200EmbeddingLoader(wespeaker.state_dict())().to(cuda_device)


def trunk(emb, x_dev, stage):
    """the map behind `stage` from the production trunk, float64 (U, T, 80) for the log-mel, (U, W, H, C) for the maps"""
    U, S = x_dev.shape
    dims = (C.c_int * 4)()
    out = np.empty(U * (S // 160) * 80 * 32, np.float32)       # the widest map: [U][T0][80][32]
    _lib.check(_lib.lib().dg_emb_debug_trunk(emb.handle, x_dev.data_ptr(), U, S, STOP[stage], out.ctypes.data, out.size, dims))
    shape = tuple(dims)[:3] if stage == "logmel" else tuple(dims)
    return out[:int(np.prod(shape))].reshape(shape).astype(np.float64)


def error(name, got, ref):
    ref = np.asarray(ref, np.float64)
    if name == "logmel":
        assert got.shape == ref.shape and np.isfinite(got).all()
        return float(np.abs(got - ref).max())
    return stage_error(got.reshape(got.shape[0], got.shape[1], -1), ref.reshape(ref.shape[0], ref.shape[1], -1))


def references(wespeaker, net64, x, w=None):
    """float64 stages, and float32 torch's for the printout"""
    return (nets.wespeaker_stages(net64, x[:, None, :].double(), None if w is None else w.double()),
            nets.wespeaker_stages(wespeaker, x[:, None, :], w))


def compare(label, emb, x_dev, ref, ref32, rows=None, stages=STAGES):
    errs = {}
    sel = (lambda a: a) if rows is None else (lambda a: a[rows])
    for name in stages:
        errs[name] = error(name, sel(trunk(emb, x_dev, name)), ref[name].numpy())
        e32 = error(name, ref32[name].double().numpy(), ref[name].numpy())
        print(f"{label:44s} {name:10s} cuda {errs[name]:.2e}   torch32 {e32:.2e}")
    return errs


def bar_of(kind, stage):
    return PINS.get(kind, {}).get(stage, BARS[stage][1])


def assert_bars(label, errs, kind="default"):
    bad = {k: (v, bar_of(kind, k)) for k, v in errs.items() if not v <= bar_of(kind, k)}
    assert not bad, f"{label}: stages beyond their bar (error, bar): {bad}"


def geometry(S):
    W = [S // 160 - 2]
    for _ in range(3):
        W.append((W[-1] - 1) // 2 + 1)
    return W


# ------------------------------------------------------------------------------------------------ shapes
# widths of the stride-2 inputs W0 / W1 / W2: 498 / 249 / 125, 298 / 149 / 75, 198 / 99 / 50, 249 / 125 / 63, 300 / 150 / 75 --
# each of the three is odd in one shape and even in another
SHAPES = [(80000, 17), (80000, 1), (80000, 3), (48000, 3), (32000, 17), (40160, 3), (48320, 1)]


@pytest.mark.parametrize("S,U", SHAPES)
def test_trunk_stages(wespeaker, net64, emb_b, cuda_device, S, U):
    x = windows("default", U, S)
    ref, ref32 = references(wespeaker, net64, x)
    W = geometry(S)
    assert emb_b.dims(S)[0] == W[3]
    errs = compare(f"default S={S} U={U}", emb_b, x.to(cuda_device), ref, ref32)
    assert ref["block15"].shape[1] == W[3] and ref["block3"].shape[1] == W[1]
    assert_bars(f"S={S} U={U}", errs)


def test_wide_batch_on_a_subset_of_items(wespeaker, net64, emb_b, cuda_device):
    """48 windows in one trunk; float64 on the first two and the last two"""
    U, rows = 48, [0, 1, 46, 47]
    x = windows("default", U)
    ref, ref32 = references(wespeaker, net64, x[rows])
    errs = compare("default S=80000 U=48, items 0 1 46 47", emb_b, x.to(cuda_device), ref, ref32, rows=rows)
    assert_bars("U=48", errs)


# ------------------------------------------------------------------------------------------------ audio
# Stages that do not meet the default stream's bar on one input, with the reason and a bound just above what was measured
# (H100 80GB HBM3, 700 W).  Every other stage of the case keeps the default bar, and every stage must be finite.
PINS = {}


def _weights(U, F, K, seed=3):
    return torch.rand((U, F, K), generator=torch.Generator().manual_seed(seed)) ** 3


@pytest.mark.parametrize("kind", list(ALL_INPUTS))
def test_stages_and_embedding_on_audio(wespeaker, net64, emb_b, cuda_device, kind):
    U = 3
    x = windows(kind, U)
    w = _weights(U, 293, 3)
    ref, ref32 = references(wespeaker, net64, x, w)
    xd = x.to(cuda_device)
    label = f"{kind} U={U}"
    errs = compare(label, emb_b, xd, ref, ref32)
    got = emb_b.forward_fused(xd, w.to(cuda_device)).cpu().numpy().astype(np.float64)
    errs["embedding"] = stage_error(got, ref["embedding"].numpy())
    print(f"{label:44s} {'embedding':10s} cuda {errs['embedding']:.2e}   "
          f"torch32 {stage_error(ref32['embedding'].double().numpy(), ref['embedding'].numpy()):.2e}")
    assert_bars(label, errs, kind)


@pytest.mark.parametrize("level", [1.0, 0.5, 0.01, 0.0, -0.3, -1.0])
def test_constant_audio_gives_the_floor(emb_b, cuda_device, level):
    """a constant window at any level in [-1, 1] has no energy after the DC removal: every bin is log(float32 eps)"""
    x = torch.full((2, 32000), level, dtype=torch.float32, device=cuda_device)
    got = trunk(emb_b, x, "logmel")
    floor = np.log(np.finfo(np.float32).eps)
    assert np.ptp(got) == 0 and abs(got[0, 0, 0] - floor) < 1e-6, (level, got.min(), got.max())


# ------------------------------------------------------------------------------------------------ embeddings
@pytest.fixture(scope="module")
def final_map(net64):
    """the float64 final map of the default stream (U = 3), in pyannote's (U, C x mel, time) pooling layout"""
    x = windows("default", 3)
    m = nets.wespeaker_stages(net64, x[:, None, :].double())["block15"]        # (U, W, H, C)
    return x, m.permute(0, 3, 2, 1).reshape(3, 256 * 10, -1)


def embed64(net64, final, w, mode="3.1"):
    pool = nets.StatsPool(mode)
    with torch.no_grad():
        return torch.stack([net64.resnet.seg_1(pool(final, w[:, :, k].double())) for k in range(w.shape[2])], dim=1).numpy()


@pytest.fixture(scope="module")
def emb_b21(wespeaker, cuda_device):
    return models.B200XVectorSincNet(wespeaker.state_dict(), pool_mode="2.1").to(cuda_device)


@pytest.mark.parametrize("frames", [293, 63], ids=["resized", "at_W3"])
@pytest.mark.parametrize("mode", ["3.1", "2.1"])
@pytest.mark.parametrize("K", [1, 3, 5])
def test_embeddings(net64, final_map, emb_b, emb_b21, cuda_device, K, mode, frames):
    x, final = final_map
    w = _weights(3, frames, K, seed=K)
    emb = emb_b if mode == "3.1" else emb_b21
    got = emb.forward_fused(x.to(cuda_device), w.to(cuda_device)).cpu().numpy().astype(np.float64)
    e = stage_error(got, embed64(net64, final, w, mode))
    print(f"{'embedding K=%d mode %s F=%d' % (K, mode, frames):44s} {'embedding':10s} cuda {e:.2e}")
    assert e <= BARS["embedding"][1]


def test_pooling_weight_edges(net64, final_map, emb_b, cuda_device):
    """the denominators of StatsPool at their edges: a speaker with no weight at all, one at the 1e-8 floor of
    OverlappedSpeechPenalty everywhere, one at the floor with one frame above it, and one frame of weight 1"""
    x, final = final_map
    t = 22
    src = int(F.interpolate(torch.arange(293.0)[None, None], size=63, mode="nearest")[0, 0, t])     # the source of frame t
    w = _weights(3, 293, 5)
    w[:, :, 0] = 0.0
    w[:, :, 1] = 1e-8
    w[:, :, 2] = 1e-8
    w[:, src, 2] = 0.5
    w[:, :, 3] = 0.0
    w[:, src, 3] = 1.0
    got = emb_b.forward_fused(x.to(cuda_device), w.to(cuda_device)).cpu().numpy().astype(np.float64)
    want = embed64(net64, final, w)
    assert np.isfinite(got).all()
    # one frame of weight 1: float64 gives that frame's values a deviation of 7e-5 |x| from 1 + 1e-8 != 1 alone; in float32
    # (pyannote's arithmetic, and this library's) 1 + 1e-8 == 1 and the deviation is exactly 0
    one = final[:, :, t]
    with torch.no_grad():
        want[:, 3] = net64.resnet.seg_1(torch.cat([one, torch.zeros_like(one)], dim=1)).numpy()
    # one frame at 0.5 over the floor: the deviation's denominator v1 - v2 / v1 + eps is 1.3e-6 as the difference of two numbers
    # near 0.5, whose float32 rounding depends on the order the 62 floor weights are summed in -- float32 torch is 1.3e-2 from
    # float64 here, this library 0.28 (H100 80GB HBM3, 700 W): bounded just above that, and finite
    bars = {2: 0.35}
    for k, name in ((0, "all-zero"), (1, "1e-8 floor"), (2, "one above"), (3, "one frame"), (4, "random")):
        e = float(np.abs(got[:, k] - want[:, k]).max()) if k == 0 else stage_error(got[:, k], want[:, k])
        print(f"{'pool weight edges':44s} {name:10s} cuda {e:.2e}")
        assert e <= bars.get(k, BARS["embedding"][1]), (name, e)


# ------------------------------------------------------------------------------------------------ buffer reuse
def test_one_handle_through_changing_shapes(wespeaker, emb_b, cuda_device):
    """the padding rings of the maps are valid for one geometry: a handle driven through other chunk lengths and batch sizes
    returns, bit for bit, what a fresh handle returns"""
    state = wespeaker.state_dict()
    for S, U in ((80000, 3), (48000, 5), (80000, 2), (80000, 5), (32000, 1)):
        x = windows("default", U, S).to(cuda_device)
        w = _weights(U, 293, 3, seed=U).to(cuda_device)
        fresh = models.B200EmbeddingLoader(state)().to(cuda_device)
        (m_used, e_used), (m_fresh, e_fresh) = [(trunk(e, x, "block15"), e.forward_fused(x, w).cpu().numpy()) for e in (emb_b, fresh)]
        assert np.array_equal(m_used, m_fresh), f"final map at S={S} U={U}"
        assert np.array_equal(e_used, e_fresh), f"embedding at S={S} U={U}"
