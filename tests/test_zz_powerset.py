"""Powerset segmentation models (pyannote/segmentation-3.0 layout; reference ``PowersetAdapter``,
``src/diart/models.py:29-39``): Linear(128, 7) -> log_softmax -> one_hot(argmax) @ mapping.

pyannote.audio is not vendored by the reference (``setup.cfg:34``) and is absent here, so ``Powerset`` is restated in
``oracle/nets.py`` from its published definition (subsets ordered by size, then as ``itertools.combinations`` yields them);
the CPU tests pin that restatement, the GPU tests compare the CUDA decoding with it.  (File name: runs last.)"""
import ctypes as C

import numpy as np
import pytest
import torch

from diart_b200 import _lib, models, synth
from oracle import nets


def test_powerset_mapping_order():
    m = nets.powerset_mapping(3, 2)
    assert m.tolist() == [[0, 0, 0], [1, 0, 0], [0, 1, 0], [0, 0, 1], [1, 1, 0], [1, 0, 1], [0, 1, 1]]
    m4 = nets.powerset_mapping(4, 2)
    assert m4.shape == (11, 4)
    assert m4[5:].tolist() == [[1, 1, 0, 0], [1, 0, 1, 0], [1, 0, 0, 1], [0, 1, 1, 0], [0, 1, 0, 1], [0, 0, 1, 1]]
    assert nets.powerset_mapping(3, 3).shape == (8, 3) and nets.powerset_mapping(2, 1).tolist() == [[0, 0], [1, 0], [0, 1]]


def test_to_multilabel_takes_the_first_maximum():
    m = nets.powerset_mapping(3, 2)
    logp = torch.full((1, 3, 7), -5.0)
    logp[0, 0, 4] = -0.1                      # {0, 1}
    logp[0, 1, 0] = -0.1                      # nobody
    logp[0, 2, 2] = logp[0, 2, 6] = -0.1      # tie between {1} and {1, 2}: argmax returns the first
    assert nets.to_multilabel(logp, m)[0].tolist() == [[1, 1, 0], [0, 0, 0], [0, 1, 0]]


def test_powerset_oracle_net_shapes():
    net = nets.make_powerset_segmentation()
    assert net.classifier.out_features == 7
    x = torch.from_numpy(synth.windows(synth.synth_audio(80000 + 8000, seed=99), 2))
    with torch.no_grad():
        y = net(x[:, None, :])
    assert y.shape == (2, 293, 3) and set(y.unique().tolist()) <= {0.0, 1.0}
    assert (y.sum(-1) <= 2).all()             # at most two speakers per frame


def test_set_powerset_argument_errors_without_gpu():
    lib = _lib.lib()
    assert lib.dg_seg_set_powerset(None, 3, 2) == -1
    assert b"dg_seg_set_powerset" in lib.dg_last_error()


@pytest.mark.gpu
def test_powerset_segmentation_matches_oracle(cuda_device):
    net = nets.make_powerset_segmentation()
    x = torch.from_numpy(synth.windows(synth.synth_audio(80000 + 8000 * 7, seed=77), 8))
    taps = {}
    with torch.no_grad():
        ref = net(x[:, None, :], taps)
    top2 = taps["log_probabilities"].topk(2, dim=-1).values
    sure = (top2[..., 0] - top2[..., 1]) > 1e-2        # frames whose arg-max survives float32-level differences of the logits
    assert sure.float().mean() > 0.9
    seg = models.B200PyanNet(net.state_dict(), powerset=(3, 2)).to(cuda_device)
    assert seg.dims(80000) == (293, 3)
    out = seg(x[:, None, :].to(cuda_device)).cpu()
    assert out.shape == ref.shape and set(out.unique().tolist()) <= {0.0, 1.0}
    assert torch.equal(out[sure], ref[sure])
    print(f"powerset: {int(sure.sum())} of {sure.numel()} frames compared, all equal")


@pytest.mark.gpu
def test_powerset_declaration_must_match_the_classifier(cuda_device):
    net = nets.make_powerset_segmentation()
    with pytest.raises((ValueError, _lib.DiartB200Error)):
        models.B200PyanNet(net.state_dict(), powerset=(4, 2)).to(cuda_device)     # 11 classes declared, 7 outputs
    plain = models.B200PyanNet(net.state_dict()).to(cuda_device)                 # not declared: 7 sigmoid outputs
    assert plain.dims(80000) == (293, 7)


# ------------------------------------------------------------------------------------------------ against float64
# The trunk of a powerset model is PyanNet's: its stages are held to the default networks' bars (tests/test_gpu_net_stages.py),
# measured on the multilabel model.  The decoded labels then equal float64's on every frame whose float64 top-two logit margin
# exceeds what the linear1 bar lets the device's logits move: |d(l_a - l_b)| <= max_{a,b} ||w_a - w_b||_1 * bar * rms(linear1),
# plus the float32 rounding of the 128-term dot products (2^-20 of max_a sum |w_a| |y|, generous).
def _powerset_case(num_speakers, max_per_frame, tie=False):
    net = nets.make_powerset_segmentation(num_speakers=num_speakers, max_per_frame=max_per_frame)
    if tie:                                   # class 6 ({1, 2}) a copy of class 2 ({1}), both favoured by the bias
        with torch.no_grad():
            net.classifier.bias[2] += 2.0
            net.classifier.weight[6] = net.classifier.weight[2]
            net.classifier.bias[6] = net.classifier.bias[2]
    return net


def _margin_bound(net, linear1):
    from test_gpu_net_stages import BARS

    w = net.classifier.weight.detach().double()
    l1 = max(float((w[a] - w[b]).abs().sum()) for a in range(w.shape[0]) for b in range(w.shape[0]) if a != b)
    rms = float(linear1.pow(2).mean().sqrt())
    dots = float((linear1.abs() @ w.abs().T).max())
    return l1 * BARS["linear1"][1] * rms + 2.0 ** -20 * dots


@pytest.mark.gpu
@pytest.mark.parametrize("num_speakers,max_per_frame,tie", [(3, 2, False), (3, 2, True), (3, 3, False), (2, 1, False)],
                         ids=["3-2", "3-2-tie", "3-3", "2-1"])
def test_powerset_stages_and_labels_match_float64(cuda_device, num_speakers, max_per_frame, tie):
    from test_gpu_net_stages import SEG_STAGES, STREAM, Hook, assert_bars, compare

    B = 5
    net = _powerset_case(num_speakers, max_per_frame, tie)
    x = torch.from_numpy(synth.windows(synth.synth_audio(80000 + 8000 * (B - 1), seed=77), B))
    ref = nets.segmentation_stages(nets.float64_copy(net), x[:, None, :].double())
    ref32 = nets.segmentation_stages(net, x[:, None, :])
    seg = models.B200PyanNet(net.state_dict(), powerset=(num_speakers, max_per_frame)).to(cuda_device)
    hook = Hook(seg, x.to(cuda_device), 8000)
    label = f"powerset ({num_speakers}, {max_per_frame}){' tie' if tie else ''}"
    errs = compare(label, hook, SEG_STAGES[:10], ref, ref32)
    assert hook.paths & STREAM
    assert_bars(label, errs)
    got = hook(10)
    assert got.shape == (B, 293, num_speakers) and set(np.unique(got).tolist()) <= {0.0, 1.0}
    logits = ref["logits"]
    distinct = logits[..., :6] if tie else logits             # a tie is not a small margin: class 6 is class 2 again
    top2 = distinct.topk(2, dim=-1).values
    margin = (top2[..., 0] - top2[..., 1]).numpy()
    bound = _margin_bound(net, ref["linear1"])
    sure = margin > bound
    print(f"{label:58s} labels: margin bound {bound:.2e}, {sure.mean():.3f} of the frames beyond it")
    assert sure.mean() > 0.9
    want = ref["scores"].numpy()
    assert np.array_equal(got[sure], want[sure])
    if tie:
        # frames where the tied pair leads: float64's logits of classes 2 and 6 are equal, and both sides take the first
        others = torch.cat([logits[..., :2], logits[..., 3:6]], dim=-1).amax(dim=-1)
        lead = ((logits[..., 2] - others).numpy() > bound)
        assert torch.equal(logits[..., 2], logits[..., 6]) and lead.mean() > 0.1
        assert np.all(got[lead] == np.array([0.0, 1.0, 0.0]))        # class 2 = {1}; `>=` in the kernel would give {1, 2}
        assert np.all(want[lead] == np.array([0.0, 1.0, 0.0]))
