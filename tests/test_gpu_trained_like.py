"""The default networks stage by stage against float64 on trained-like weights (tests/trained_like.py): mean-dominated
InstanceNorm inputs (R1) and TDNN5 channels (R2) and near-dead BatchNorm (R3), at S = 80 000 in both sinc forms (fused MaxPool3
statistics and fused TDNN5 pooling) and at S = 48 000 (the un-fused paths).

Matmul stages keep the measure and the bars of tests/test_gpu_net_stages.py.  R1 at mean / std >= 1000 goes past what a
float32 evaluation resolves and is held to the bound of an error model instead: the float32 map and the 22-bit operand planes
keep a mean-dominated value to about 2^-22 of its mean, so the channel's normalised output carries 2^-22 x (mean / std) per
element, and every later stage mixes it in; the stage maximum is held to 2^-18 x (mean / std).  The factor 16 over the
per-element figure is the one the default bars carry (tests/test_gpu_net_stages.py): 4 for a maximum over 10^5 .. 10^7 elements
against an RMS, 4 from the l1 / l2 norm ratio of the weight rows that mix the channel into the next stage (tdnn0, whose 60
inputs include it, sits at 13 x the per-element figure).  Measured (NVIDIA H100 80GB
HBM3, 700 W limit): at 1000, 3.1e-3 at tdnn0 and 2.2e-3 at lstm2 (float32 torch, printed beside every stage, 2.9e-3 and
5.5e-4); at 10^4, 1.7e-2 at tdnn0 (float32 torch 2.2e-2).  The R3 probe channel carries almost all of TDNN1's energy, so TDNN1 is measured without it and the probe channel on
its own scale.
Statistics are checked per channel: the InstanceNorm rstd of the mean-dominated channels (the ratio of the normalised maps'
deviations over time, after undoing LeakyReLU and beta) and every pooled standard deviation above a floor, each relative to
float64.  The bar of a fused statistic is 4 x the error of the robust path on the same weights (the un-fused InstanceNorm at
S = 48 000, POOLED_PLAIN for POOLED_FUSED), with a floor of 1e-5: the float32 maps and outputs round each value to 6e-8 of it,
and a deviation of a mean-dominated channel to 2^-24 x mean / std, which stays under 1e-5 after averaging over the frames."""
import numpy as np
import pytest
import torch

import trained_like as tl
from diart_b200 import models, synth
from oracle import nets
from test_gpu_net_stages import (BARS, EMB_STAGES, POOLED_FUSED, POOLED_PLAIN, POOLF, POOL3, SEG_STAGES, STREAM, Hook, compare,
                                 stage_error)

pytestmark = pytest.mark.gpu

FLOOR = 1e-5
STD_FLOOR = 2.0 ** -16          # pooled deviations below this share of |mean| are not resolved by a float32 map
FORMS = [(80000, 8000), (80000, 0), (48000, 8000)]


@pytest.fixture(scope="module")
def x80():
    torch.set_num_threads(16)
    return tl.windows()


_CACHE = {}


def cached(key, fn):
    if key not in _CACHE:
        _CACHE[key] = fn()
    return _CACHE[key]


def run(label, state, is_seg, S, hop, device, w=None, stages=None):
    """float64 and float32 torch stages of `state` and the CUDA hook's -> ({stage: error}, hook, ref64)"""
    x = tl.windows(samples=S)
    net = tl.segmentation(state) if is_seg else tl.embedding(state)
    fn = nets.segmentation_stages if is_seg else nets.embedding_stages
    args = () if is_seg or w is None else (w,)
    ref = cached((label, S, "64"), lambda: fn(nets.float64_copy(net), x[:, None, :].double(), *[a.double() for a in args]))
    ref32 = cached((label, S, "32"), lambda: fn(net, x[:, None, :], *args))
    cuda = models.B200PyanNet(state) if is_seg else models.B200XVectorSincNet(state)
    cuda = cuda.to(device)
    hook = Hook(cuda, x.to(device), hop, None if w is None else w.to(device))
    stages = stages or (SEG_STAGES if is_seg else EMB_STAGES)
    errs = compare(f"{label} S={S} {'stream' if hop else 'window'}", hook, stages, ref, ref32)
    assert bool(hook.paths & STREAM) == (hop > 0)
    assert bool(hook.paths & POOL3) == (S == 80000)
    return errs, hook, ref


def over(errs, bars):
    return {k: (v, bars.get(k, BARS[k][1])) for k, v in errs.items() if not v <= bars.get(k, BARS[k][1])}


# ------------------------------------------------------------------------------------------------ R1
def _linear(y, beta):
    """undo LeakyReLU(0.01) and the InstanceNorm beta: gamma (v - mean) rstd"""
    return np.where(y > 0, y, y / 0.01) - beta


def rstd_errors(got, ref, state, c, row):
    """relative error of the InstanceNorm rstd of channel `row` of sinc_norm{c}, per window"""
    beta = state[f"sincnet.norm1d.{c}.bias"][row].item()
    g, r = _linear(got[:, :, row], beta), _linear(ref[:, :, row], beta)
    return np.abs(g.std(axis=1) / r.std(axis=1) - 1.0)


@pytest.mark.parametrize("net", ["seg", "emb"])
@pytest.mark.parametrize("ratio", tl.LADDER)
def test_r1_mean_dominated_instancenorm(x80, cuda_device, net, ratio):
    base = synth.segmentation_state() if net == "seg" else synth.embedding_state()
    state = cached(("r1", net, ratio), lambda: tl.r1_state(base, ratio, x80))
    stages = {}
    for S, hop in FORMS:
        errs, hook, ref = run(f"R1 {net} {ratio:.0f}", state, net == "seg", S, hop, cuda_device)
        stat = {}
        for c, (row, _) in tl.R1_ROWS.items():
            stat[c] = float(rstd_errors(hook(c), ref[f"sinc_norm{c}"].numpy(), state, c, row).max())
            print(f"R1 {net} mean/std {ratio:7.0f} S={S} {'stream' if hop else 'window'}: conv{c} rstd error {stat[c]:.2e}")
        stages[(S, hop)] = (errs, stat)
        # float32 cannot resolve the deviation of a channel 1000 x its spread from its mean better than the model's bound
        model = {k: max(BARS[k][1], 2.0 ** -18 * ratio) for k in errs} if ratio >= 1000 else {}
        assert not over(errs, model), (S, hop, over(errs, model))
    robust = stages[(48000, 8000)][1]
    for S, hop in FORMS[:2]:
        for c, e in stages[(S, hop)][1].items():
            assert e <= max(4 * robust[c], FLOOR), (S, hop, c, e, robust[c])


# ------------------------------------------------------------------------------------------------ R2
@pytest.mark.parametrize("K", [3, 4])
def test_r2_mean_dominated_pooling(x80, cuda_device, K):
    state = cached(("r2",), lambda: tl.r2_state(synth.embedding_state(), x80))
    w = tl.pool_weights(K=K)
    x = tl.windows()
    ref = cached(("r2 pool", K), lambda: nets.embedding_stages(nets.float64_copy(tl.embedding(state)), x[:, None, :].double(),
                                                                 w.double())["stats_pool"].numpy())
    cuda = models.B200XVectorSincNet(state).to(cuda_device)
    hook = Hook(cuda, x.to(cuda_device), 8000, w.to(cuda_device))
    mean, std = ref[:, :, :1500], ref[:, :, 1500:]
    resolved = std > STD_FLOOR * np.abs(mean)
    errs = {}
    for stage, name in ((POOLED_FUSED, "fused"), (POOLED_PLAIN, "plain")):
        got = hook(stage).reshape(tl.B, K, 3000)
        assert bool(hook.paths & POOLF) == (name == "fused")
        assert np.isfinite(got).all()
        rel = np.abs(got[:, :, 1500:] / np.where(resolved, std, 1.0) - 1.0) * resolved
        errs[name] = rel
        e_mean = stage_error(got[:, :, :1500], mean)
        print(f"R2 K={K} {name:6s} mean {e_mean:.2e}, std (all resolved entries) {rel.max():.2e}")
        assert e_mean <= BARS["stats_pool"][1]
        for row, ratio, b in tl.r2_rows():
            print(f"R2 K={K} {name:6s} row {row} b {b:+.0f} mean/std {ratio:7.0f}: std error {rel[:, :, row].max():.2e}")
    bar = max(4 * errs["plain"].max(), FLOOR)
    assert errs["fused"].max() <= bar, (errs["fused"].max(), bar)


def test_r2_one_frame_weight_on_mean_dominated_channels(x80, cuda_device):
    """the edge of pool_finalize's resolution clamp with pivots far from the BatchNorm shift: one frame of weight 1, the R2
    channels at mean / std up to 10^4.  float64 gives a deviation of 5.8e-5 |x| from 1 + 1e-8 != 1 alone (in float32
    1 + 1e-8 == 1 and the deviation is 0); both poolings give 0 or that, and the fused mean is the two-pass pooling's (the
    frame's float32 value) to float32 rounding: the pivots and tile sums are exact or rounded to 2^-24 of the deviation"""
    state = cached(("r2",), lambda: tl.r2_state(synth.embedding_state(), x80))
    x, K = tl.windows(), 3
    w = torch.zeros((tl.B, 293, K))
    w[:, 100, :] = 1.0
    ref = cached(("r2 one frame",), lambda: nets.embedding_stages(nets.float64_copy(tl.embedding(state)), x[:, None, :].double(),
                                                                   w.double())["stats_pool"].numpy())
    hook = Hook(models.B200XVectorSincNet(state).to(cuda_device), x.to(cuda_device), 8000, w.to(cuda_device))
    rows = [r for r, _, _ in tl.r2_rows()]
    means = {}
    for stage, name in ((POOLED_FUSED, "fused"), (POOLED_PLAIN, "plain")):
        got = hook(stage).reshape(tl.B, K, 3000)
        assert bool(hook.paths & POOLF) == (name == "fused") and np.isfinite(got).all()
        mean, std = got[:, :, :1500], got[:, :, 1500:]
        means[name] = mean
        e_mean = stage_error(mean, ref[:, :, :1500])
        d_std = np.abs(std - ref[:, :, 1500:])
        e_std = (d_std[:, :, rows] / np.abs(ref[:, :, rows])).max()          # the R2 rows, on the scale of their own mean
        e_all = d_std.max() / np.abs(ref[:, :, :1500]).max()                 # every channel (test_pooling_single_frame_weight)
        print(f"R2 one frame {name:6s}: mean {e_mean:.2e}, R2 rows |std - float64| / |mean| {e_std:.2e}, all {e_all:.2e}")
        assert e_mean <= BARS["stats_pool"][1]
        assert np.all(std >= 0) and e_std <= 1e-4 and e_all <= 1e-4
    # the R2 rows relative to their own mean; every channel on the scale of the largest mean (a channel whose mean is near 0
    # keeps 2^-24 of the BatchNorm shift it is taken around, as the parent's sums did)
    diff = np.abs(means["fused"] - means["plain"])
    d_rows = (diff[:, :, rows] / np.abs(means["plain"][:, :, rows])).max()
    d_all = diff.max() / np.abs(means["plain"]).max()
    print(f"R2 one frame: fused mean vs two-pass mean, R2 rows {d_rows:.2e} relative, all {d_all:.2e}")
    assert d_rows <= 2.0 ** -21 and d_all <= 2.0 ** -21


# ------------------------------------------------------------------------------------------------ R3
def test_r3_near_dead_batchnorm(x80, cuda_device):
    state = cached(("r3",), lambda: tl.r3_state(synth.embedding_state(), x80))
    for S, hop in FORMS:
        errs, _, _ = run("R3 near-dead BN", state, False, S, hop, cuda_device)
        assert not over(errs, {}), (S, hop, over(errs, {}))


@pytest.mark.parametrize("peak", [2.0 ** 14, 2.0 ** 15])
def test_r3_activations_at_the_fp16_edge(x80, cuda_device, peak):
    """a TDNN1 channel whose activations reach 2^14 / 2^15 stays inside the hi plane's range (saturation starts above 65504)"""
    state = cached(("r3 probe", peak), lambda: tl.r3_probe_state(synth.embedding_state(), x80, peak))
    errs, hook, ref = run(f"R3 probe {peak:.0f}", state, False, 80000, 8000, cuda_device)
    i, ch = tl.R3_PROBE
    got, want = hook(4 + i), ref[f"tdnn{i}"].numpy()
    assert abs(float(np.abs(want[:, :, ch]).max()) / peak - 1) < 1e-6
    errs[f"tdnn{i}"] = stage_error(np.delete(got, ch, axis=2), np.delete(want, ch, axis=2))
    probe = stage_error(got[:, :, ch:ch + 1], want[:, :, ch:ch + 1])
    print(f"R3 probe {peak:.0f}: tdnn{i} without the probe channel {errs[f'tdnn{i}']:.2e}, the probe channel {probe:.2e}")
    assert probe <= BARS[f"tdnn{i}"][1]
    assert not over(errs, {}), over(errs, {})
