"""The trained-like weight regimes (tests/trained_like.py) on the CPU: every regime reaches its stated condition in float64, and
a float32 emulation of the fused statistics, in the kernels' summation order, predicts what the one-pass sums lose on the
mean-dominated rungs of R1 and R2 and what the pivoted sums (the current kernels) keep.

Emulated order (gemm_tc.cu, TC_MAXPOOL3 and TC_POOL): per tile, four row groups -- thread rg sums rows rg, rg + 4, ... (MaxPool3)
or rows 32 rg .. 32 rg + 31 (pooling) in float32 -- added ((g0 + g1) + g2) + g3 in float32, the tiles of an item in float64
(sincnet.cu: instnorm_finalize, heads.cu: pool_finalize)."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

import trained_like as tl
from diart_b200 import synth
from oracle import nets

STAT_BAR = 1e-3          # relative error of a standard deviation that the fused statistics must stay under


@pytest.fixture(scope="module")
def x():
    torch.set_num_threads(16)
    return tl.windows()


# ------------------------------------------------------------------------------------------------ float32 emulation
f32 = np.float32


def instnorm_std(v, tile_frames, pivoted):
    """v (T,) float32 pooled pre-bias values of one (window, channel) -> the std the fused InstanceNorm statistics give"""
    T = len(v)
    tiles = []
    for t0 in range(0, T, tile_frames):
        tile = v[t0:t0 + tile_frames]
        p = tile[0] if pivoted else f32(0)
        g = []
        for rg in range(4):
            s1 = s2 = f32(0)
            for e in tile[rg::4]:
                d = f32(e - p)
                s1 = f32(s1 + d)
                s2 = f32(np.float64(d) * d + s2)          # fmaf: one rounding
            g.append((s1, s2))
        s1 = f32(f32(f32(g[0][0] + g[1][0]) + g[2][0]) + g[3][0])
        s2 = f32(f32(f32(g[0][1] + g[1][1]) + g[2][1]) + g[3][1])
        tiles.append((float(p), len(tile), float(s1), float(s2)))
    if not pivoted:
        m = sum(t[2] for t in tiles) / T
        return np.sqrt(max(sum(t[3] for t in tiles) / T - m * m, 0.0))
    m = sum(n * p + s1 for p, n, s1, _ in tiles) / T
    return np.sqrt(max(sum(s2 + 2 * (p - m) * s1 + n * (p - m) ** 2 for p, n, s1, s2 in tiles) / T, 0.0))


def pooled_std(d, w, item_rows, T, eps, pivoted):
    """d (B, item_rows) float32 deviations from the BatchNorm shift (zero weight past T), w (B, item_rows) float32 weights ->
    per window the weighted std the fused TDNN5 pooling gives (pyannote StatsPool, mode 3.1); pivoted: each tile around the
    average of d at two of the item's valid rows where they sit far from 0 next to their difference, else around 0"""
    Bn = d.shape[0]
    dd, ww = d.reshape(-1), w.reshape(-1)
    out = []
    for b in range(Bn):
        r0, r1 = b * item_rows, (b + 1) * item_rows
        tiles = []
        for mt in range(r0 // 128, (r1 - 1) // 128 + 1):
            lo, hi = max(r0, mt * 128), min(r1, mt * 128 + 128)
            nv = max(0, min(hi, r0 + T) - lo)
            p = f32(0)
            if pivoted and nv:
                pa, pb = dd[lo], dd[lo + nv // 2]
                p = f32(f32(0.5) * f32(pa + pb)) if abs(f32(pa + pb)) > 16 * abs(f32(pa - pb)) else f32(0)
            g = []
            for rg in range(4):
                a0, a1 = max(lo, mt * 128 + 32 * rg), min(hi, mt * 128 + 32 * rg + 32)
                s1 = s2 = f32(0)
                for r in range(a0, a1):
                    e = f32(dd[r] - p)
                    a = f32(ww[r] * e)
                    s1 = f32(s1 + a)
                    s2 = f32(np.float64(a) * e + s2)
                g.append((s1, s2))
            s1 = f32(f32(f32(g[0][0] + g[1][0]) + g[2][0]) + g[3][0])
            s2 = f32(f32(f32(g[0][1] + g[1][1]) + g[2][1]) + g[3][1])
            tiles.append((float(p), float(np.sum(ww[lo:hi], dtype=np.float64)), float(s1), float(s2)))
        v2 = float(np.sum(ww[r0:r1].astype(np.float64) ** 2))
        v1 = float(f32(f32(np.sum(ww[r0:r1])) + f32(eps)))         # launch_pool_weights: float32
        if pivoted:     # shifted to the first tile's pivot, in double
            P = tiles[0][0]
            W = sum(wt for _, wt, _, _ in tiles)
            s1P = sum(s1 + wt * (p - P) for p, wt, s1, _ in tiles)
            s2P = sum(s2 + (p - P) * (2 * s1 + wt * (p - P)) for p, wt, s1, s2 in tiles)
            dq = (s1P + W * P) / v1 - P
            num = s2P - 2 * dq * s1P + dq * dq * W
            s2c = sum(t[3] for t in tiles)
        else:
            s1t, s2t = sum(t[2] for t in tiles), sum(t[3] for t in tiles)
            dm = s1t / v1
            num = s2t - 2 * dm * s1t + dm * dm * (v1 - eps)
            s2c = s2t
        num = 0.0 if (num < s2c * 2.0 ** -20 or num < 0) else num
        out.append(np.sqrt(num / (v1 - v2 / v1 + eps)))
    return np.array(out)


def ref_pooled_std(d, w, eps):
    d, w = d.astype(np.float64), w.astype(np.float64)
    v1 = w.sum(axis=1) + eps
    mean = (d * w).sum(axis=1) / v1
    return np.sqrt(((d - mean[:, None]) ** 2 * w).sum(axis=1) / (v1 - (w ** 2).sum(axis=1) / v1 + eps))


# ------------------------------------------------------------------------------------------------ R1
@pytest.mark.parametrize("net", ["emb", "seg"])
def test_r1_reaches_its_ladder_and_the_one_pass_sums_break(x, net):
    base = synth.embedding_state() if net == "emb" else synth.segmentation_state()
    for ratio in tl.LADDER:
        state = tl.r1_state(base, ratio, x)
        facts = tl.r1_facts(state, x)
        pooled = tl.pooled_prenorm(state, x)
        for c, (row, _) in tl.R1_ROWS.items():
            assert np.all((facts[c] > ratio / 1.5) & (facts[c] < ratio * 1.5)), (net, c, ratio, facts[c])
            # the other channels keep the synthetic weights' own regime (mean / std about 6)
            others = np.delete(np.abs(tl.ratio_of(pooled[c])), row, axis=1)
            assert np.median(others) < 20, (net, c, np.median(others))
            v = pooled[c][:, row, :].numpy().astype(np.float32)
            tile_frames = {1: 37, 2: 37}[c]            # tiles of 111 un-pooled rows at S = 80 000 (items of 2664 / 888 rows)
            want = v.astype(np.float64).std(axis=1)
            old = np.array([instnorm_std(vb, tile_frames, False) for vb in v])
            new = np.array([instnorm_std(vb, tile_frames, True) for vb in v])
            e_old, e_new = np.abs(old / want - 1).max(), np.abs(new / want - 1).max()
            print(f"R1 {net} conv{c} mean/std {ratio:7.0f}: one-pass std error {e_old:.2e}, pivoted {e_new:.2e}")
            assert e_new < 1e-5
            if ratio <= 10:
                assert e_old < STAT_BAR / 10
            if ratio >= 1000:
                assert e_old > STAT_BAR


# ------------------------------------------------------------------------------------------------ R2
def test_r2_reaches_its_ladder_and_the_one_pass_sums_break(x):
    w = tl.pool_weights()
    state = tl.r2_state(synth.embedding_state(), x)
    facts = tl.r2_facts(state, x, w)
    net = nets.float64_copy(tl.embedding(state))
    t5 = nets.embedding_stages(net, x[:, None, :].double())["tdnn4"].numpy()            # (B, T, 1500)
    T = t5.shape[1]
    item_rows = 296                                                                      # trunk rows per item at S = 80 000 (T = 279)
    wr = F.interpolate(w.permute(0, 2, 1), size=T, mode="nearest").permute(0, 2, 1).numpy().astype(np.float32)
    shift = state["tdnns.14.bias"].numpy() - state["tdnns.14.running_mean"].numpy() * (
        state["tdnns.14.weight"].numpy() / np.sqrt(state["tdnns.14.running_var"].numpy() + tl.EPS_BN))
    for row, ratio, b in tl.r2_rows():
        r = np.abs(facts[row])
        assert np.all((r > ratio / 1.5) & (r < ratio * 1.5)), (row, ratio, b, r)
        d = np.zeros((tl.B, item_rows), np.float32)
        d[:, :T] = (t5[:, :, row].astype(np.float32) - np.float32(shift[row]))
        for k in range(w.shape[2]):
            wk = np.zeros((tl.B, item_rows), np.float32)
            wk[:, :T] = wr[:, :, k]
            want = ref_pooled_std(d, wk, 1e-8)
            old = pooled_std(d, wk, item_rows, T, 1e-8, False)
            new = pooled_std(d, wk, item_rows, T, 1e-8, True)
            e_old, e_new = np.abs(old / want - 1).max(), np.abs(new / want - 1).max()
            print(f"R2 row {row} b {b:+.0f} mean/std {ratio:7.0f} speaker {k}: one-pass std error {e_old:.2e}, pivoted {e_new:.2e}")
            assert e_new < 1e-5
            if ratio <= 10:
                assert e_old < STAT_BAR / 10
            if ratio >= 1000:
                assert e_old > STAT_BAR


# ------------------------------------------------------------------------------------------------ R3
def test_r3_near_dead_batchnorm(x):
    facts = tl.bn_facts(tl.r3_state(synth.embedding_state(), x), x)
    for i, f in facts.items():
        print(f"R3 tdnn{i}", f)
        assert f["zero_var"] > 0 and f["min_var"] == 0.0                 # channels with running_var exactly 0
        assert f["max_gain"] > 1000 and f["max_gamma"] <= 4.0            # gamma / sqrt(eps) reached, gamma within [0.2, 4]
        assert f["max_act"] < 65504                                      # a realistic regime stays inside the fp16 range


@pytest.mark.parametrize("peak", [2.0 ** 14, 2.0 ** 15])
def test_r3_probe_reaches_the_fp16_edge(x, peak):
    f = tl.bn_facts(tl.r3_probe_state(synth.embedding_state(), x, peak), x)[tl.R3_PROBE[0]]
    assert abs(f["max_act"] / peak - 1) < 1e-6 and f["zero_var"] >= 1


def test_r3_near_dead_batchnorm_wespeaker():
    base = nets.make_wespeaker().state_dict()
    state = tl.r3_wespeaker_state(base)
    f = tl.wespeaker_bn_facts(state, tl.windows(3))
    print("R3 WeSpeaker", f)
    assert f["zero_var"] > 0 and f["min_var"] == 0.0
    assert f["max_gain"] > 1000 and f["max_gamma"] <= 4.0
    assert f["max_act"] < 65504
    # only BatchNorm parameters and the producing convolutions change
    assert all(k.endswith((".weight", ".running_mean", ".running_var")) for k in state if not torch.equal(state[k], base[k]))
