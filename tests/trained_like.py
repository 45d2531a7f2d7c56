"""Trained-like weight regimes for the float64 stage tests: deterministic transforms of the synthetic state dicts
(diart_b200.synth) that reach the numerical regimes trained checkpoints can reach and uniform random-init weights do not.
Each regime changes only what it targets and returns the float64 facts that show its condition was reached
(tests/test_trained_like_host.py asserts them, tests/test_gpu_trained_like.py runs the CUDA path on the same weights).

R1  mean-dominated InstanceNorm inputs of SincNet conv1 / conv2: an input channel made exactly constant (InstanceNorm gamma 0,
    beta = LEVEL) is read by one output row with weight C_READ on every tap; the row's other weights are scaled so that the
    pooled (pre-bias) output has mean / std = the rung.  MaxPool commutes with adding a constant and with positive scaling, so
    the ratio is set exactly for the calibration windows.
R2  mean-dominated TDNN5 channels: rows scaled by eps with bias +-2 sit at leaky(b) * scale + shift with a spread set by eps.
R3  near-dead BatchNorm in TDNN1-5 and in every BatchNorm of WeSpeaker ResNet34: channels whose pre-activation barely moves
    (the producing row scaled by delta, or exactly constant) with running statistics that match it (running_var down to exactly
    0), gamma in [0.2, 4].  Because the statistics match, BatchNorm renormalises these channels and activations stay moderate
    (float64 peak 693 in the TDNNs); the other side of a near-dead BatchNorm -- the gain gamma / sqrt(eps) = 316 gamma applied
    to a channel that does move -- is reached by one probe channel of TDNN1, scaled so that its float64 activation peaks at
    2^14 / 2^15 (the fp16 planes saturate above 65504).
"""
from __future__ import annotations

import numpy as np
import torch
import torch.nn.functional as F

from diart_b200 import synth
from oracle import nets

S, B, HOP = 80000, 4, 8000
LADDER = (10.0, 100.0, 1000.0, 10000.0)
LEVEL, C_READ = 64.0, 0.5            # R1: the constant channel's value and the weight that reads it (both exact in fp16)
R1_ROWS = {1: (1, 0), 2: (3, 2)}     # conv c: (mean-dominated output row, constant input channel of its input)
R2_BIAS = (2.0, -2.0)                # both slopes of the LeakyReLU
R2_FIRST_ROW = 40                    # R2 rows: R2_FIRST_ROW + 2 * rung + sign
R3_PROBE = (1, 7)                    # R3 probe: TDNN index, channel
EPS_BN = 1e-5


def windows(n=B, samples=S, hop=HOP, seed=77):
    """n consecutive windows of the default synthetic stream (tests/test_gpu_net_stages.py: make_windows("default"))"""
    stream = synth.synth_audio(samples + hop * (n - 1), seed=seed).astype(np.float64).astype(np.float32)
    return torch.from_numpy(synth.windows(stream, n, chunk=samples, step=hop))


def segmentation(state):
    return nets._load(nets.PyanNet(num_speakers=3), state)


def embedding(state):
    return nets._load(nets.XVectorSincNet(), state)


def pool_weights(n=B, frames=293, K=3, seed=3):
    return torch.rand((n, frames, K), generator=torch.Generator().manual_seed(seed)) ** 3


# ------------------------------------------------------------------------------------------------ R1
def pooled_prenorm(state, x, prefix="sincnet."):
    """float64 (B, C, T) pooled, pre-bias outputs of SincNet conv1 and conv2 -- what the InstanceNorm statistics see"""
    net = nets.float64_copy(embedding({**synth.embedding_state(), **{k: v for k, v in state.items() if k.startswith(prefix)}}))
    maps = nets.sincnet_stages(net.sincnet, x[:, None, :].double())
    with torch.no_grad():
        return {c: F.max_pool1d(F.conv1d(maps[f"sinc_norm{c - 1}"].transpose(1, 2), state[f"{prefix}conv1d.{c}.weight"].double()), 3, 3)
                for c in (1, 2)}


def ratio_of(v):
    """mean / std over time of every (window, channel) of a (B, C, T) map"""
    return (v.mean(dim=2) / v.std(dim=2, unbiased=False)).numpy()


def r1_state(base, ratio, x):
    """`base` with conv1 row 1 and conv2 row 3 mean-dominated at `ratio` (pooled mean / std, median over the windows)"""
    s = {k: v.clone() for k, v in base.items()}
    for c, (row, ch) in R1_ROWS.items():
        s[f"sincnet.norm1d.{c - 1}.weight"][ch] = 0.0
        s[f"sincnet.norm1d.{c - 1}.bias"][ch] = LEVEL
        w = s[f"sincnet.conv1d.{c}.weight"]
        w[row, ch, :] = 0.0
        rest = pooled_prenorm(s, x)[c][:, row, :]          # the row without the constant channel
        mu_big = C_READ * LEVEL * w.shape[2]
        m, sd = float(rest.mean(dim=1).median()), float(rest.std(dim=1, unbiased=False).median())
        w[row] *= mu_big / (ratio * sd - m)                 # (mu_big + k m) / (k sd) = ratio
        w[row, ch, :] = C_READ
    return s


def r1_facts(state, x):
    p = pooled_prenorm(state, x)
    return {c: ratio_of(p[c])[:, row] for c, (row, _) in R1_ROWS.items()}


# ------------------------------------------------------------------------------------------------ R2
def r2_rows():
    return [(R2_FIRST_ROW + 2 * i + j, ratio, b) for i, ratio in enumerate(LADDER) for j, b in enumerate(R2_BIAS)]


def r2_state(base, x):
    """TDNN5 rows at leaky(b) * scale + shift with mean / std = every rung, for both signs of b"""
    s = {k: v.clone() for k, v in base.items()}
    net = nets.float64_copy(embedding(base))
    h = nets.embedding_stages(net, x[:, None, :].double())["tdnn3"]            # TDNN5's input (B, T, 512)
    W = s["tdnns.12.weight"]
    for row, ratio, b in r2_rows():
        z = h @ W[row, :, 0].double()
        mz, sz = float(z.mean()), float(z.std(unbiased=False))
        # BatchNorm mean and shift 0: the channel is k leaky(eps z + b), mean / std = (b + eps mz) / (eps sz) = ratio
        s["tdnns.14.running_mean"][row] = 0.0
        s["tdnns.14.bias"][row] = 0.0
        W[row] *= b / (ratio * sz * np.sign(b) - mz)
        s["tdnns.12.bias"][row] = b
    return s


def r2_facts(state, x, w):
    net = nets.float64_copy(embedding(state))
    pooled = nets.embedding_stages(net, x[:, None, :].double(), w.double())["stats_pool"].numpy()    # (B, K, 3000)
    rows = [r for r, _, _ in r2_rows()]
    return {r: pooled[:, :, r] / pooled[:, :, 1500 + r] for r in rows}


# ------------------------------------------------------------------------------------------------ R3
def r3_state(base, x, seed=11):
    """in every TDNN BatchNorm, a third of the channels near-dead: the producing row scaled by delta = 10^U(-4, -1) (a sixth of
    them by 0: exactly constant), running mean / var = the channel's own float64 statistics (so running_var spans 0 .. 1e-2 x
    the live channels'), gamma U(0.2, 4) everywhere"""
    g = torch.Generator().manual_seed(seed)
    s = {k: v.clone() for k, v in base.items()}
    for i in range(5):
        n = s[f"tdnns.{3 * i}.weight"].shape[0]
        dead = torch.randperm(n, generator=g)[: n // 3]
        delta = 10.0 ** (-4 + 3 * torch.rand(len(dead), generator=g))
        delta[: len(dead) // 6] = 0.0
        s[f"tdnns.{3 * i}.weight"][dead] *= delta[:, None, None]
        s[f"tdnns.{3 * i + 2}.weight"] = 0.2 + 3.8 * torch.rand(n, generator=g)
        # running statistics of the pre-BatchNorm activation, layer by layer on the modified net
        net = nets.float64_copy(embedding(s))
        with torch.no_grad():
            h = nets.sincnet_stages(net.sincnet, x[:, None, :].double())["sinc_norm2"].transpose(1, 2)
            for j in range(3 * i + 2):
                h = net.tdnns[j](h)
        s[f"tdnns.{3 * i + 2}.running_mean"][dead] = h.mean(dim=(0, 2))[dead].float()
        s[f"tdnns.{3 * i + 2}.running_var"][dead] = h.var(dim=(0, 2), unbiased=False)[dead].float()
    return s


def r3_probe_state(base, x, peak):
    """TDNN1 channel R3_PROBE[1] with running_var 0, mean 0, beta 0 and gamma set so that its float64 activation peaks at `peak`"""
    i, ch = R3_PROBE
    s = {k: v.clone() for k, v in base.items()}
    for n, v in (("running_var", 0.0), ("running_mean", 0.0), ("bias", 0.0), ("weight", 1.0)):
        s[f"tdnns.{3 * i + 2}.{n}"][ch] = v
    act = nets.embedding_stages(nets.float64_copy(embedding(s)), x[:, None, :].double())[f"tdnn{i}"][:, :, ch]
    s[f"tdnns.{3 * i + 2}.weight"][ch] = peak / float(act.abs().max())
    return s


def bn_facts(state, x):
    """per TDNN: the largest |activation|, the smallest running_var, the channels with running_var exactly 0, the largest
    BatchNorm gain gamma / sqrt(running_var + eps)"""
    out = nets.embedding_stages(nets.float64_copy(embedding(state)), x[:, None, :].double())
    facts = {}
    for i in range(5):
        rv, g = state[f"tdnns.{3 * i + 2}.running_var"].double(), state[f"tdnns.{3 * i + 2}.weight"].double()
        facts[i] = {"max_act": float(out[f"tdnn{i}"].abs().max()), "min_var": float(rv.min()), "zero_var": int((rv == 0).sum()),
                    "max_gain": float((g.abs() / torch.sqrt(rv + EPS_BN)).max()), "max_gamma": float(g.abs().max())}
    return facts


def wespeaker(state):
    return nets._load(nets.WeSpeakerResNet34(), state)


def _producer(bn):
    """the convolution whose output a WeSpeaker BatchNorm normalises"""
    if bn.endswith("shortcut.1"):
        return bn[:-1] + "0"
    return bn.replace(".bn", ".conv")


def r3_wespeaker_state(base, seed=17):
    """every BatchNorm of WeSpeaker ResNet34 with a third of its channels near-dead: the producing convolution's filter scaled by
    delta = 10^U(-4, -1) (a sixth of them by 0: the channel is exactly 0, running_var exactly 0) and the running statistics
    scaled with it (the convolutions have no bias: the channel's mean scales by delta, its variance by delta^2), gamma
    U(0.2, 4) everywhere"""
    g = torch.Generator().manual_seed(seed)
    s = {k: v.clone() for k, v in base.items()}
    for bn in sorted(k[: -len(".running_var")] for k in s if k.endswith(".running_var")):
        n = s[bn + ".weight"].shape[0]
        dead = torch.randperm(n, generator=g)[: n // 3]
        delta = 10.0 ** (-4 + 3 * torch.rand(len(dead), generator=g))
        delta[: len(dead) // 6] = 0.0
        s[_producer(bn) + ".weight"][dead] *= delta[:, None, None, None]
        s[bn + ".running_mean"][dead] *= delta
        s[bn + ".running_var"][dead] *= delta ** 2
        s[bn + ".weight"] = 0.2 + 3.8 * torch.rand(n, generator=g)
    return s


def wespeaker_bn_facts(state, x):
    """over all WeSpeaker BatchNorms: the smallest running_var, the channels with running_var exactly 0, the largest gain and
    gamma; the largest float64 |activation| of the stem and the 16 blocks"""
    rv = torch.cat([v.double() for k, v in state.items() if k.endswith(".running_var")])
    gam = torch.cat([state[k[: -len("running_var")] + "weight"].double() for k in state if k.endswith(".running_var")])
    out = nets.wespeaker_stages(nets.float64_copy(wespeaker(state)), x[:, None, :].double())
    return {"min_var": float(rv.min()), "zero_var": int((rv == 0).sum()), "max_gamma": float(gam.abs().max()),
            "max_gain": float((gam.abs() / torch.sqrt(rv + EPS_BN)).max()),
            "max_act": max(float(out[k].abs().max()) for k in out if k != "logmel")}
